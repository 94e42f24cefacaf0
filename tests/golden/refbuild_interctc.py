"""refbuild.model_yaml with intermediate CTC in the encoder and, optionally, no decoder.  Test infrastructure.  Chains whatever
refbuild.model_yaml is installed when install() runs.

cfg keys (ints, as fixtures store cfg as int64): ic_a, ic_b -- the listed layers (1-based; 0 = not listed), ic_cond -- self-conditioning on
(1) or off (0), no_decoder -- 1 for a CTC-only model without a decoder (the LibriSpeech-100 train_conformer_scctc.yaml recipe).
"""
import refbuild


def interctc_conf(cfg):
    return dict(interctc_layer_idx=[v for v in (cfg.get("ic_a", 0), cfg.get("ic_b", 0)) if v],
                interctc_use_conditioning=bool(cfg.get("ic_cond", 0)))


def wrap(model_yaml):
    def with_interctc(cfg):
        y = model_yaml(cfg)
        y["encoder_conf"] = dict(y["encoder_conf"], **interctc_conf(cfg))
        y["model_conf"] = dict(y["model_conf"], interctc_weight=0.3)
        if cfg.get("no_decoder", 0):
            y["decoder"], y["decoder_conf"] = None, {}
            y["model_conf"]["ctc_weight"] = 1.0
        return y
    return with_interctc


def install(monkeypatch=None):
    """Route refbuild.model_yaml (and with it refbuild.build_reference, gpu_util.speech2text) through wrap(); with a pytest monkeypatch
    the change is undone after the test."""
    if monkeypatch is None:
        refbuild.model_yaml = wrap(refbuild.model_yaml)
    else:
        monkeypatch.setattr(refbuild, "model_yaml", wrap(refbuild.model_yaml))
