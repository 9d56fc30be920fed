"""CPU tests of the drop-in boundary: the C-ABI library builds, loads without a CUDA driver, exports every symbol
that include/ctrl_adapter_b200.h declares, and fails loudly (no silent fallback) when no GPU is present."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from ctrl_adapter_b200 import _lib, build
    build.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "ctrl_adapter_b200.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(ca_\w+)\s*\(", hdr, flags=re.M))
    assert len(declared) >= 20
    from ctrl_adapter_b200 import _lib
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(raw, name), f"{name} declared in the header but not exported"
    assert declared == set(_lib.SIGNATURES), "ctypes SIGNATURES and header declarations differ"


def test_abi_version_and_struct_sizes(lib):
    from ctrl_adapter_b200 import _lib
    assert lib.ca_abi_version() == 1
    # the ctypes mirror must have the C layout: compile-time sizes are checked against gcc's view of the header
    import subprocess, tempfile
    src = '#include <stdio.h>\n#include "ctrl_adapter_b200.h"\nint main(){printf("%zu %zu", sizeof(ca_gemm_desc), sizeof(ca_attention_desc));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        out = subprocess.check_output([exe]).decode().split()
    assert int(out[0]) == ctypes.sizeof(_lib.GemmDesc)
    assert int(out[1]) == ctypes.sizeof(_lib.AttentionDesc)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_fails_loudly_without_gpu(lib):
    from ctrl_adapter_b200 import _lib, ops
    assert lib.ca_device_ok() != 0
    assert b"CUDA" in lib.ca_last_error() or b"device" in lib.ca_last_error()
    with pytest.raises(ValueError, match="no CPU path"):
        ops.linear(torch.zeros(4, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    d = _lib.GemmDesc()
    assert lib.ca_gemm(ctypes.byref(d), None) == 1  # CA_ERR_INVALID, with a message
    assert len(lib.ca_last_error()) > 0


def test_gemm_rejects_blend_with_fp32_output(lib):
    """The fp32 epilogue has no AlphaBlender term: ca_gemm refuses the combination instead of dropping the blend.
    Argument validation runs before any tensor map is encoded, so placeholder pointers and no device suffice."""
    from ctrl_adapter_b200 import _lib
    d = _lib.GemmDesc()
    d.nsrc, d.ntaps = 1, 1
    d.box[0], d.box[1], d.box[2], d.box[3] = 128, 1, 1, 1
    d.a[0] = d.w = d.out = d.blend_src = d.blend_alpha = 256  # never dereferenced
    d.a_channels[0] = d.a_c_len[0] = d.w_k_per_tap = 64
    d.a_dims[0] = d.a_dims[1] = d.a_dims[2] = d.a_dims[3] = 1
    d.out_dims[0] = d.out_dims[1] = d.out_dims[2] = d.out_dims[3] = 1
    d.w_rows = d.n_out = 64
    d.out_fp32 = 1
    assert lib.ca_gemm(ctypes.byref(d), None) == 3  # CA_ERR_UNSUPPORTED
    assert b"blend" in lib.ca_last_error()


_P = 256  # placeholder device / host pointer: validation fails before anything is dereferenced
_INVALID_CALLS = [  # entry point, arguments with one out of range, what the message must name
    ("ca_silu", (_P, 12, _P, None), b"n (12)"),
    ("ca_add", (_P, _P, 12, _P, None), b"n (12)"),
    ("ca_upsample2x", (_P, 1, 4, 4, 12, _P, None), b"c (12)"),
    ("ca_avgpool", (_P, 1, 10, 8, 8, 4, 4, _P, None), b"oh, ow"),
    ("ca_router_weights", (_P, _P, 1, 33, _P, None), b"nexperts"),
    ("ca_router_merge", (_P, _P, 9, 64, _P, None), b"nactive"),
    ("ca_softmax_rows", (_P, 1, 6, _P, None), b"cols (6)"),
    ("ca_layernorm", (_P, 4, 12, 1e-5, _P, _P, None, 0, None, _P, None), b"c (12)"),
    ("ca_groupnorm_stats", (_P, 40, None, 0, 1, 16, 32, _P, None), b"groups (32)"),
    ("ca_cfg_euler_v", (_P, _P, _P, 64, _P, 0, 16, _P, 1, _P, _P, None), b"frames"),
    ("ca_i2vgen_latent_encoder", (_P, 1, 33, 16, 8, _P, _P, None), b"frames"),
    ("ca_temporal_attention", (_P, _P, _P, 1, 33, 16, 1, 0.125, 64, _P, None), b"frames"),
    ("ca_frame_conv_small", (_P, 1, 4, 16, 8, 5, 3, _P, None, _P, None), b"cin"),
]


@pytest.mark.parametrize("name,args,names", _INVALID_CALLS, ids=[c[0] for c in _INVALID_CALLS])
def test_entry_point_rejects_invalid_argument(lib, name, args, names):
    """Every entry point checks its arguments before any CUDA call: an out-of-range one returns CA_ERR_INVALID (Python
    raises ValueError) with a message naming it, with or without a GPU."""
    assert getattr(lib, name)(*args) == 1
    assert names in lib.ca_last_error()


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "ctrl_adapter_b200")
    for f in os.listdir(pkg):
        if f.endswith(".py"):
            src = open(os.path.join(pkg, f)).read()
            assert "oracle" not in src.replace("# oracle", ""), f"{f} references the oracle"
