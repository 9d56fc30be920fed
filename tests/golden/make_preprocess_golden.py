"""Generates tests/golden/reference_preprocess_golden.json by running the REAL reference function
``_resize_with_antialiasing`` (/root/reference/utils/utils_svd.py, which imports only torch and numpy) on seeded images
in fp32 on CPU: the anti-aliased resize the SVD pipeline applies before its CLIP image encoder
(svd/pipelines/svd_controlnet_adapter_pipeline.py:177-179).  tests/test_vae_encoder_cpu.py pins the package's
restatement (ctrl_adapter_b200.pipelines._resize_with_antialiasing) against these fingerprints.

Kept apart from make_golden.py so that reference_golden.json is not regenerated.
Run in the build container only (needs /root/reference):   python tests/golden/make_preprocess_golden.py
"""
import importlib.util
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.weights import fingerprint  # noqa: E402

spec = importlib.util.spec_from_file_location("ref_utils_svd", "/root/reference/utils/utils_svd.py")
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

CASES = {  # name: (input shape [n, 3, H, W], output size, generator seed); inputs = 2 * rand - 1
    "576x1024_to_224": ((1, 3, 576, 1024), (224, 224), 1),
    "320x320_to_224": ((2, 3, 320, 320), (224, 224), 2),
    "704x1280_to_224": ((1, 3, 704, 1280), (224, 224), 3),
}
out = {"_meta": {"reference": "utils/utils_svd.py _resize_with_antialiasing @ /root/reference", "torch": torch.__version__,
                 "input": "torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2 - 1, fp32 CPU"},
       "resize_with_antialiasing": {}}
with torch.no_grad():
    for name, (shape, size, seed) in CASES.items():
        x = torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2 - 1
        y = ref._resize_with_antialiasing(x, size)
        out["resize_with_antialiasing"][name] = {"input_shape": list(shape), "size": list(size), "seed": seed,
                                                 "out": fingerprint(y)}
        print(name, tuple(y.shape))
path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_preprocess_golden.json")
with open(path, "w") as f:
    json.dump(out, f)
print("wrote", path, os.path.getsize(path), "bytes")
