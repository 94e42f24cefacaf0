"""Plugging the espnet_b200 classes into an UNMODIFIED espnet2 installation (the reference's registries and scorer protocol).

``register()`` derives, for every espnet_b200 module class, a subclass that also inherits the reference's abstract base
(AbsFrontend / AbsNormalize / AbsEncoder / AbsDecoder + BatchScorerInterface, as ``ClassChoices`` type-checks, espnet2/train/class_choices.py:33-54)
and adds it to the registries of ``espnet2.tasks.asr`` (asr.py:96-206) under a ``b200_`` name.  A training config that says
``frontend: b200_default``, ``normalize: b200_utterance_mvn``, ``encoder: b200_conformer``, ``decoder: b200_transformer`` then builds the CUDA
modules through the reference's own ``ASRTask.build_model`` and decodes through the reference's own ``Speech2Text`` / ``BatchBeamSearch``
(device="cuda"), the decoder being driven through ``batch_score`` / ``select_state``.  ``espnet2`` must be importable; nothing in the
espnet_b200 hot path imports this module.  See INTEGRATION.md.
"""
import espnet_b200

NAMES = {"frontend": {"b200_default": "DefaultFrontend"},
         "normalize": {"b200_utterance_mvn": "UtteranceMVN", "b200_global_mvn": "GlobalMVN"},
         "encoder": {"b200_conformer": "ConformerEncoder", "b200_transformer": "TransformerEncoder",
                     "b200_contextual_block_conformer": "ContextualBlockConformerEncoder",
                     "b200_contextual_block_transformer": "ContextualBlockTransformerEncoder", "b200_e_branchformer": "EBranchformerEncoder",
                     "b200_branchformer": "BranchformerEncoder"},
         "decoder": {"b200_transformer": "TransformerDecoder"}}


def _derive(name, base, *abcs, extra=None):
    ns = {"__doc__": f"espnet_b200.{name} registered under the reference's {', '.join(a.__name__ for a in abcs)}", "__module__": __name__}
    ns.update(extra or {})
    return type(name, (base,) + abcs, ns)


def register():
    """Returns {registry name: {choice name: class}} of what was added (idempotent)."""
    import espnet2.tasks.asr as asr_task
    from espnet2.asr.decoder.abs_decoder import AbsDecoder
    from espnet2.asr.encoder.abs_encoder import AbsEncoder
    from espnet2.asr.frontend.abs_frontend import AbsFrontend
    from espnet2.layers.abs_normalize import AbsNormalize
    from espnet2.legacy.nets.scorer_interface import BatchScorerInterface

    def _no_training_forward(self, hs_pad, hlens, ys_in_pad, ys_in_lens):
        raise NotImplementedError("espnet_b200.TransformerDecoder is an inference scorer (batch_score); the training forward is not on this path")

    bases = {"frontend": (AbsFrontend,), "normalize": (AbsNormalize,), "encoder": (AbsEncoder,), "decoder": (AbsDecoder, BatchScorerInterface)}
    added = {}
    for reg, names in NAMES.items():
        choices = getattr(asr_task, f"{reg}_choices")
        for choice, cls_name in names.items():
            if choice not in choices.classes:
                extra = {"forward": _no_training_forward} if reg == "decoder" else None
                choices.classes[choice] = _derive(cls_name, getattr(espnet_b200, cls_name), *bases[reg], extra=extra)
            added.setdefault(reg, {})[choice] = choices.classes[choice]
    return added


def ctc_prefix_scorer(ctc, eos):
    """espnet_b200.CTCPrefixScorer as an instance of the reference's BatchPartialScorerInterface (what its BeamSearch type-checks)."""
    from espnet2.legacy.nets.scorer_interface import BatchPartialScorerInterface

    from .ctc import CTCPrefixScorer

    cls = type("CTCPrefixScorer", (CTCPrefixScorer, BatchPartialScorerInterface), {"__module__": __name__})
    return cls(ctc, eos)
