"""lfm_b200.inpaint_metrics on the H100 (`-m gpu`) with the stand-in detector of tests/test_inpaint_metrics_host.py on cuda:0:
batched features against one-image calls, the metrics against the restated reference run on the CPU, and the downstream
readme's two steps end to end: the inpainting command line, then its scoring on the files it wrote."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from lfm_b200 import inpaint_metrics as im
from tests.test_gpu_vae_encoder import write_dataset
from tests.test_inpaint_metrics_host import load_detector, save_detector, write_set
from tests.tools import inpaint_metrics_oracle as oracle

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:`torch.jit:DeprecationWarning")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def test_batched_features_match_one_image_calls(dev, tmp_path):
    """fp32 stand-in (the real detector is fp32): cuDNN may take other algorithms for a batch of 9 than for one image."""
    gen, gt = write_set(tmp_path, n=30, size=(48, 48))
    det = load_detector(save_detector(tmp_path / "det.pt", dims=64, dtype=torch.float32), dev)
    files, _, sizes = im.image_pairs(gen, gt)
    tf32 = torch.backends.cudnn.allow_tf32
    feats, stats = im.detector_features(det, files, sizes, 9, dev)
    assert torch.backends.cudnn.allow_tf32 == tf32                   # restored after the feature pass
    assert feats.device.type == "cuda" and feats.dtype == torch.float32 and feats.shape == (30, 64)
    assert stats.s1.device.type == "cuda" and stats.s1.dtype == torch.float64 and stats.n == 30
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            one = torch.cat([det(torch.from_numpy(im.read_image(f))[None].to(dev), return_features=True) for f in files])
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert float((feats - one).norm() / one.norm()) <= 1e-5


def test_metrics_match_cpu_oracle(dev, tmp_path):
    gen, gt = write_set(tmp_path, n=40, seed=4)
    path = save_detector(tmp_path / "det.pt")
    got = im.inpainting_metrics(gen, gt, load_detector(path, dev), batch_size=16, device=dev)
    want = oracle.inpainting_metrics(gen, gt, load_detector(path, "cpu"))
    assert abs(got[0] - want[0]) <= 1e-6 * want[0]
    assert got[1:] == want[1:]


def test_inpainting_then_scoring_end_to_end(dev, tmp_path):
    gt, masks = write_dataset(tmp_path, 16)
    out = tmp_path / "run"
    gen = subprocess.run([sys.executable, os.path.join(ROOT, "test_flow_latent_inpainting.py"), "--synthetic_init", "1",
                          "--synthetic_vae", "1", "--num_images", "16", "--batch_size", "8", "--method", "euler",
                          "--step_size", "0.25", "--gt_dir", gt, "--mask_dir", masks, "--out_dir", str(out),
                          "--num_workers", "0", "--device", "cuda:0"], cwd=ROOT, capture_output=True, text=True)
    assert gen.returncode == 0, gen.stderr[-4000:]
    gen_dir = str(out / "inpainting_generated_samples" / "celeba_256")
    assert sorted(os.listdir(gen_dir), key=lambda s: int(s[:-4])) == [f"{i}.jpg" for i in range(16)]

    path = save_detector(tmp_path / "det.pt", dims=8)
    result = tmp_path / "fid_pids_uids.txt"
    score = subprocess.run([sys.executable, "-m", "lfm_b200.inpaint_metrics", gen_dir, gt, "--detector", path,
                            "--out", str(result), "--batch-size", "8", "--device", "cuda:0"],
                           cwd=ROOT, capture_output=True, text=True)
    assert score.returncode == 0, score.stderr[-4000:]
    line = result.read_text()
    assert score.stdout.splitlines()[-1] == line
    m = re.fullmatch(r"fid: (\d+\.\d{4}), pids: (\d\.\d{4}), uids: (\d\.\d{4})", line)
    assert m, line

    fid_value, pids, uids = oracle.inpainting_metrics(gen_dir, gt, load_detector(path, "cpu"))
    assert abs(float(m.group(1)) - fid_value) <= 5e-5 + 1e-6 * fid_value
    assert (m.group(2), m.group(3)) == ("%.4f" % pids, "%.4f" % uids)
    assert fid_value > 0
