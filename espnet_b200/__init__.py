"""espnet_b200: H100-native (sm_90a) implementation of ESPnet2's Speech2Text inference hot path.

Public surface mirrors the reference classes on that path (see SURVEY.md section 8b):
Speech2Text, ESPnetASRModel, DefaultFrontend, UtteranceMVN, ConformerEncoder, CTC,
TransformerDecoder, BatchBeamSearch, Hypothesis, TooShortUttError (+ GlobalMVN, the output-side text classes, and the
TransformerEncoder of the next scope row, the EBranchformerEncoder and the BranchformerEncoder, the RNN family's VGGRNNEncoder, RNNEncoder and RNNDecoder; CTCPrefixScorer and TransformerDecoder.batch_score implement the reference's scorer protocol,
``espnet_b200.integration.register()`` adds the classes to the reference's registries).
All compute goes through the C-ABI CUDA library ``libespnet_b200.so`` (include/espnet_b200.h).
"""
from .asr_inference import (ESPnetASRModel, Speech2Text, build_model, build_model_from_file, decoder_choices,  # noqa: F401
                            encoder_choices, frontend_choices, normalize_choices)
from .branchformer_encoder import BranchformerEncoder  # noqa: F401
from .ctc import CTC, CTCPrefixScorer  # noqa: F401
from .decoder import TransformerDecoder  # noqa: F401
from .e_branchformer_encoder import EBranchformerEncoder  # noqa: F401
from .encoder import ConformerEncoder  # noqa: F401
from .errors import TooShortUttError  # noqa: F401
from .frontend import DefaultFrontend, GlobalMVN, LogMel, UtteranceMVN  # noqa: F401
from .rnn_decoder import RNNDecoder  # noqa: F401
from .rnn_encoder import RNNEncoder, VGGRNNEncoder  # noqa: F401
from .lm import SequentialRNNLM, TransformerLM, build_lm_from_file  # noqa: F401
from .search import BatchBeamSearch, Hypothesis  # noqa: F401
from .search_online import BatchBeamSearchOnline, LengthBonus  # noqa: F401
from .asr_inference_streaming import Speech2TextStreaming  # noqa: F401
from .streaming_encoder import ContextualBlockConformerEncoder, ContextualBlockTransformerEncoder  # noqa: F401
from .text import TokenIDConverter, build_tokenizer  # noqa: F401
from .transformer_encoder import TransformerEncoder  # noqa: F401

__version__ = "0.1.0"
