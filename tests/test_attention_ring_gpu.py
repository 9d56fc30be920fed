"""pytest -m gpu: attention at KV tile counts that stress the kernel's K / V rings and its pipelined schedule (the
softmax of tile j + 1 runs while P V of tile j is on the tensor cores), against check_attention's fp32 reference and
tolerances (tests/kernel_checks.py)."""
import pytest
import torch

from tests import kernel_checks as kc

pytestmark = pytest.mark.gpu

# (b, heads, lq, lk, d, ramp)
CASES = [
    # an odd number of KV tiles (3) with a ragged last tile of 1 / 44 keys
    (2, 5, 300, 257, 64, 0.0),
    (2, 5, 257, 300, 64, 3.0),
    # more KV tiles than twice the ring depth: 11 tiles through 4 slots (head dim 128), 6 through 2 (head dim 192)
    (1, 4, 300, 1300, 128, 4.0),
    (1, 4, 300, 700, 160, 4.0),
]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device is visible (there is no CPU fallback to test)")
    from ctrl_adapter_b200 import _lib
    _lib.check(_lib.load().ca_device_ok(), "ca_device_ok")


@pytest.mark.parametrize("b,heads,lq,lk,d,ramp", CASES, ids=[f"lk{c[3]}_d{c[4]}" for c in CASES])
def test_attention_kv_tiles(b, heads, lq, lk, d, ramp):
    kc.RESULTS.clear()
    rec = kc.check_attention(b, heads, lq, lk, d, ramp=ramp)
    print(rec)
    assert rec["ok"], rec
