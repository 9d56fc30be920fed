"""GPU: every case of the ABI domain sweep (tests/abi_domain.py) at full size on the real kernels, under the guarded
recorder of tests/launch_checks.py (float64 verdicts, NaN / pattern guard bands around every operand, bit-identical
replay, no byte outside the argument views changed).  Each case's first launch runs under torch.profiler (a kernel trace
only): the template arguments of the kernels it launched must be exactly the name-visible branches the case predicts,
and a branch counts as reached only where its kernel was observed.  -s prints one row per case, a per-entry-point
summary, the kernel instantiations observed and the branches that are run-time switches (predicted only), and the
file's peak device memory."""
import time

import pytest
import torch

from tests import abi_domain as ad
from tests import launch_checks as lc

pytestmark = pytest.mark.gpu


def test_abi_domain_sweep():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    cs = ad.cases()
    with torch.no_grad(), ad.KernelTrace() as tr, lc.Recorder() as rec:
        res = ad.run_cases(cs, "cuda", rec, trace=tr)
    problems, reached, inst = ad.observed_dispatch(cs, tr.seen)
    print("\n" + ad.summary(cs, res))
    print(ad.dispatch_summary(reached, inst))
    print(f"\n{len(cs)} cases in {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 20:.0f} MiB")
    bad = ad.failures(res)
    assert not bad, "\n".join(f"{label}: {r.why}" for label, r in bad[:8])
    assert not problems, "\n".join(problems[:8])
    assert ad.expected_branches() <= reached, sorted(ad.expected_branches() - reached)
