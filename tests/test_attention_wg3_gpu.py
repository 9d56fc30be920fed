"""pytest -m gpu: head-dim-64 attention around ca_attention's choice between 192-row query tiles (three consumer
warpgroups) and 128-row tiles, at query tile tails, ragged and long KV rings, shared K / V contexts, fused-QKV strided
views and nearly one-hot rows, against the fp32 / fp64 references and tolerances of tests/kernel_checks.py."""
import pytest
import torch

from tests import kernel_checks as kc

pytestmark = pytest.mark.gpu

# (b, heads, lq, lk, ramp): lq 191, 192 and 383 take 192-row tiles, 193 and 1024 128-row tiles (tail padding rule);
# lk 129 leaves a 1-key last tile, lk 1300 runs 11 KV tiles through the 4-slot ring, ramp 40 gives nearly one-hot rows
# whose scaled logits span several hundred log2 units
CASES = [
    (2, 3, 191, 300, 0.0),
    (2, 3, 192, 129, 0.0),
    (2, 3, 193, 257, 0.0),
    (1, 4, 383, 1300, 0.0),
    (2, 5, 1024, 1024, 0.0),
    (1, 2, 4096, 4096, 0.0),
    (2, 3, 383, 700, 40.0),
    (1, 2, 4096, 1100, 40.0),
]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")


@pytest.mark.parametrize("b,heads,lq,lk,ramp", CASES, ids=[f"lq{c[2]}_lk{c[3]}_ramp{c[4]:g}" for c in CASES])
def test_attention_d64(b, heads, lq, lk, ramp):
    kc.RESULTS.clear()
    rec = kc.check_attention(b, heads, lq, lk, 64, ramp=ramp)
    print(rec)
    assert rec["ok"], rec


@pytest.mark.parametrize("b,heads,l", [(1, 2, 16384), (2, 3, 383), (2, 2, 193)], ids=["l16384", "l383", "l193"])
def test_attention_d64_fused_qkv(b, heads, l):
    kc.RESULTS.clear()
    rec = kc.check_attention_fused_qkv(b, heads, l, 64)
    print(rec)
    assert rec["ok"], rec


@pytest.mark.parametrize("b,lq,lk,div", [(4, 383, 300, 2), (6, 1024, 1300, 3), (2, 191, 129, 2)],
                         ids=["lq383_lk300_div2", "lq1024_lk1300_div3", "lq191_lk129_div2"])
def test_attention_d64_cross_kv(b, lq, lk, div):
    kc.RESULTS.clear()
    rec = kc.check_attention_cross_kv(b, 2, lq, lk, 64, kv_batch_div=div)
    print(rec)
    assert rec["ok"], rec
