"""refbuild.model_yaml with the encoder's input layer taken from cfg["input_layer"] (conv2d2 / conv2d6 / conv2d8; default conv2d).  Test
infrastructure.  Chains whatever refbuild.model_yaml is installed when install() runs (e.g. refbuild_ebf's E-Branchformer yaml)."""
import refbuild


def wrap(model_yaml):
    def with_input_layer(cfg):
        y = model_yaml(cfg)
        if "input_layer" in cfg:
            y["encoder_conf"] = dict(y["encoder_conf"], input_layer=cfg["input_layer"])
        return y
    return with_input_layer


def install(monkeypatch=None):
    """Route refbuild.model_yaml (and with it refbuild.build_reference, gpu_util.speech2text / random_weights) through wrap(); with a
    pytest monkeypatch the change is undone after the test."""
    if monkeypatch is None:
        refbuild.model_yaml = wrap(refbuild.model_yaml)
    else:
        monkeypatch.setattr(refbuild, "model_yaml", wrap(refbuild.model_yaml))
