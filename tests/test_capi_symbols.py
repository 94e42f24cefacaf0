"""The C-ABI library loads on a CPU-only box and exports every symbol include/espnet_b200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "espnet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(espb_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_bound_symbols():
    from espnet_b200 import lib

    assert _header_symbols() == sorted(lib.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    from espnet_b200 import lib

    if not os.path.exists(lib.LIB_PATH):
        import __graft_entry__ as g

        g.build()
    handle = ctypes.CDLL(lib.LIB_PATH)
    for sym in _header_symbols():
        assert hasattr(handle, sym), sym
    handle.espb_abi_version.restype = ctypes.c_int
    from espnet_b200 import lib as _l

    assert handle.espb_abi_version() == _l.ABI_VERSION == 7


def test_binding_arity_matches_header():
    """Every ctypes signature in lib._SIGS has as many arguments as the C prototype in include/espnet_b200.h (incl. the stream)."""
    from espnet_b200 import lib

    src = open(os.path.join(ROOT, "include", "espnet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = dict(re.findall(r"\bint\s+(espb_[a-z0-9_]+)\s*\(([^;]*?)\)\s*;", src, flags=re.S))
    for name, sig in lib._SIGS.items():
        assert name in protos, name
        params = [a for a in protos[name].split(",") if a.strip() and a.strip() != "void"]
        assert len(params) == len(sig), (name, len(params), len(sig))
        assert "cudaStream_t" in params[-1], name
        for c_arg, ct in zip(params, sig):   # pointers bind to c_void_p, scalars to the matching ctypes scalar
            is_ptr = "*" in c_arg or "cudaStream_t" in c_arg
            binds_ptr = ct is ctypes.c_void_p or issubclass(ct, ctypes._Pointer)
            assert is_ptr == binds_ptr, (name, c_arg, ct)
            if not is_ptr:
                want = ctypes.c_longlong if "long long" in c_arg else ctypes.c_float if "float" in c_arg else ctypes.c_int
                assert ct is want, (name, c_arg, ct)


def test_ops_refuse_cpu_tensors():
    """No CPU fallback: the product path fails loudly instead of computing on the host."""
    import torch

    import espnet_b200

    fe = espnet_b200.DefaultFrontend()
    with pytest.raises((AssertionError, RuntimeError)):
        fe(torch.zeros(1, 4000), torch.tensor([4000]))
    with pytest.raises(RuntimeError):
        espnet_b200.Speech2Text(asr_model=None, device="cpu")


def test_state_dict_names_match_reference_fixture():
    import argparse
    import sys

    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import refbuild
    from golden_util import load

    import espnet_b200

    for case in ("tiny", "small"):
        z, cfg, w = load(case)
        model = espnet_b200.build_model(argparse.Namespace(**refbuild.model_yaml(cfg)))
        model.load_state_dict(w, strict=True)


def test_unsupported_configs_are_rejected():
    import espnet_b200

    with pytest.raises(NotImplementedError):
        espnet_b200.ConformerEncoder(80, 256, rel_pos_type="legacy", macaron_style=True)
    with pytest.raises(NotImplementedError):
        espnet_b200.DefaultFrontend(n_fft=400)


def test_transformer_encoder_state_dict_names_match_reference_fixture():
    """Next scope row (SURVEY.md 8f-1): a reference TransformerEncoder checkpoint loads by name (strict)."""
    import numpy as np
    import torch

    import espnet_b200

    z = np.load(os.path.join(ROOT, "tests", "golden", "transformer_enc.npz"))
    cfg = dict(zip(z["cfg_keys"].tolist(), z["cfg_vals"].tolist()))
    w = {k[len("w:encoder."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    enc = espnet_b200.TransformerEncoder(80, output_size=cfg["d_model"], attention_heads=cfg["heads"], linear_units=cfg["ff"],
                                         num_blocks=cfg["layers"])
    enc.load_state_dict(w, strict=True)
    assert espnet_b200.encoder_choices["transformer"] is espnet_b200.TransformerEncoder
    with pytest.raises(NotImplementedError):
        espnet_b200.TransformerEncoder(80, 64, input_layer="linear")


# Entry points the GPU tests reach only through a wrapper, each with the test that runs it.
COVERED_THROUGH_WRAPPER = {
    "espb_gemm_f32": "tests/test_gpu_gemm.py::test_linear_plain",                                   # ops.gemm / ops.linear
    "espb_abi_version": "tests/test_capi_symbols.py::test_library_exports_every_declared_symbol",    # lib.load
    "espb_last_error": "tests/test_gpu_encoder_kernels.py::test_layernorm_refuses_D",               # lib.check on a refused call
}


def test_every_entry_point_has_a_gpu_test():
    """Each espb_* entry point of the header is named in a GPU test file (test_gpu_*.py, or a file with GPU-marked tests), or is on
    COVERED_THROUGH_WRAPPER with a test that exists."""
    import glob

    gpu_src = ""
    for f in sorted(glob.glob(os.path.join(ROOT, "tests", "*.py"))):
        src = open(f).read()
        if os.path.basename(f).startswith("test_gpu_") or "pytest.mark.gpu" in src:
            gpu_src += src
    named = {s for s in _header_symbols() if re.search(r"\b" + s + r"\b", gpu_src)}
    uncovered = sorted(set(_header_symbols()) - named - set(COVERED_THROUGH_WRAPPER))
    assert not uncovered, f"entry points no GPU test calls: {uncovered}"
    for sym, test in COVERED_THROUGH_WRAPPER.items():
        assert sym in _header_symbols(), f"{sym} is not in the header any more"
        path, name = test.split("::")
        assert re.search(r"^def " + name + r"\(", open(os.path.join(ROOT, path)).read(), flags=re.M), f"{sym}: {test} does not exist"
