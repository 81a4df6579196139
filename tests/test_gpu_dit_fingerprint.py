"""The DiT forward and an Euler run with CFG, in the bf16 and the FP8 mode, give the bytes recorded by
scripts/make_dit_golden.py (tests/golden/dit_fingerprint.npz): host-side changes to the DiT must keep its numerics bit for bit."""
import importlib.util
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def load_recipe():
    spec = importlib.util.spec_from_file_location("make_dit_golden", os.path.join(ROOT, "scripts", "make_dit_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_dit_bit_identical_to_the_recorded_fingerprint(dev):
    g = np.load(os.path.join(ROOT, "tests", "golden", "dit_fingerprint.npz"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if int(g["num_sms"]) != sms:
        pytest.skip(f"fingerprint recorded with {int(g['num_sms'])} SMs ({g['device']}); the GEMM tile plan differs on {sms}")
    got = load_recipe().fingerprint(dev)
    assert sorted(k for k in got) == sorted(k for k in g.files if k.endswith(("_sha256", "_sub")))
    for k, v in got.items():
        if k.endswith("_sub"):
            assert np.array_equal(v, g[k]), k
        else:
            assert v == str(g[k]), k
