"""CPU: ca_attention accepts exactly the positive, finite softmax scales (its kernel takes the row max on the raw
scores, which is the max of the scaled scores only for scale > 0) and rejects every other one with CA_ERR_INVALID and
a message naming the scale.  The real library through ctypes, without a GPU, on tests/abi_domain.py's placeholder
arguments: a scale inside the domain gets through validation and fails at the launch (CA_ERR_CUDA)."""
import json
import os
import subprocess
import sys

import pytest

INSIDE = [0.125, 1e-30, 1e30]
OUTSIDE = [0.0, -0.0, -0.125, float("inf"), float("-inf"), float("nan"), 3e38]

_CHILD = """
import json, sys
from ctrl_adapter_b200 import _lib
from tests import abi_domain as ad
lib = _lib.load()
out = []
for s in json.loads(sys.argv[1]):
    st = ad.c_call(lib, "ca_attention", ad.with_value("ca_attention", "scale", float(s)))
    out.append([st, lib.ca_last_error().decode(errors="replace")])
json.dump(out, sys.stdout)
"""


@pytest.fixture(scope="module")
def statuses():
    from ctrl_adapter_b200 import build
    build.build()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    scales = [repr(s) for s in INSIDE + OUTSIDE]
    r = subprocess.run([sys.executable, "-c", _CHILD, json.dumps(scales)], cwd=root, env=env, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return dict(zip(scales, json.loads(r.stdout)))


@pytest.mark.parametrize("scale", INSIDE, ids=[repr(s) for s in INSIDE])
def test_scale_inside(statuses, scale):
    st, msg = statuses[repr(scale)]
    assert st == 2, f"scale {scale} returned {st} ({msg}), expected CA_ERR_CUDA at the launch"


@pytest.mark.parametrize("scale", OUTSIDE, ids=[repr(s) for s in OUTSIDE])
def test_scale_outside(statuses, scale):
    st, msg = statuses[repr(scale)]
    assert st == 1 and "scale" in msg, f"scale {scale} returned {st} ({msg}), expected CA_ERR_INVALID"
