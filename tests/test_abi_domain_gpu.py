"""GPU: every case of the ABI domain sweep (tests/abi_domain.py) at full size on the real kernels, under the guarded
recorder of tests/launch_checks.py (float64 verdicts, NaN / pattern guard bands around every operand, bit-identical
replay, no byte outside the argument views changed), and every predicted dispatch branch reached.  -s prints one row
per case and a per-entry-point summary."""
import pytest
import torch

from tests import abi_domain as ad
from tests import launch_checks as lc

pytestmark = pytest.mark.gpu


def test_abi_domain_sweep():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cs = ad.cases()
    with torch.no_grad(), lc.Recorder() as rec:
        res = ad.run_cases(cs, "cuda", rec)
    print("\n" + ad.summary(cs, res))
    bad = ad.failures(res)
    assert not bad, "\n".join(f"{label}: {r.why}" for label, r in bad[:8])
    reached = set().union(*(c.branches for c in cs))
    assert ad.expected_branches() <= reached, sorted(ad.expected_branches() - reached)
