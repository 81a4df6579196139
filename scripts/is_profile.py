"""Cost of the Inception Score on cuda:0, next to the card's name and power limit.

1. Images/s of the IS pass (``prepare_tf1`` + trunk + ``fc`` + softmax, ``inception_score.inception_probs``) and of the
   FID pass (``FIDInception.prepare`` + trunk) at batch 200 on 256 x 256 uint8 images, seeded stand-in weights (the cost
   does not depend on the values).  CUDA events, best of several repeats.
2. The ``--compute_fid`` generation loop of a small configuration (DiT-B/2, 256 pixels, Euler with 20 steps, batch 64,
   256 images, synthetic weights, no files written) with and without ``--compute_is``, alternating, host clock around
   ``cli.main`` (it synchronises: the scores are read back).

python scripts/is_profile.py [OUT_DIR]      (prints one JSON line per part; with OUT_DIR also writes OUT_DIR/is_profile.json)"""
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lfm_b200 import cli, fid  # noqa: E402
from lfm_b200 import inception_score as lis  # noqa: E402

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True, timeout=30).stdout.strip()
rec = {"gpu": q or torch.cuda.get_device_name(0)}
print(json.dumps(rec), flush=True)


def best_ms(fn, reps=5, iters=3):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / iters)
    return best


B = 200
net = fid.FIDInception({**fid.synthetic_inception_state_dict(1), **fid.synthetic_fc_state_dict(1)}, with_logits=True).to(dev)
u8 = (torch.rand(B, 256, 256, 3, generator=torch.Generator().manual_seed(0)) * 255).to(torch.uint8).to(dev)
is_ms = best_ms(lambda: lis.inception_probs(net, u8, B))
fid_ms = best_ms(lambda: net(u8))
resize_ms = best_ms(lambda: lis.prepare_tf1(u8), iters=20)
rec["network_pass"] = {"batch": B, "side": 256, "is_ms": round(is_ms, 2), "is_images_per_s": round(B / is_ms * 1e3, 1),
                       "fid_ms": round(fid_ms, 2), "fid_images_per_s": round(B / fid_ms * 1e3, 1),
                       "prepare_tf1_ms": round(resize_ms, 3)}
print(json.dumps(rec["network_pass"]), flush=True)
del u8
torch.cuda.empty_cache()

tmp = tempfile.mkdtemp()
stat = os.path.join(tmp, "stat.npy")
feats = np.random.RandomState(0).rand(64, 2048)
np.save(stat, {"mu": feats.mean(0), "sigma": np.cov(feats, rowvar=False)}, allow_pickle=True)
loop = ["--model_type", "DiT-B/2", "--image_size", "256", "--num_in_channels", "4", "--num_classes", "1",
        "--label_dropout", "0.", "--method", "euler", "--step_size", "0.05", "--synthetic_init", "3", "--synthetic_vae", "2",
        "--device", "cuda:0", "--dataset", "custom", "--exp", "p", "--compute_fid", "--synthetic_inception", "1", "--no_save",
        "--batch_size", "64", "--n_sample", "256", "--real_img_dir", stat, "--out_dir", tmp]
times = {"fid": [], "fid_is": []}
for rep in range(3):
    for name, extra in (("fid", []), ("fid_is", ["--compute_is", "--is_splits", "4"])):
        t0 = time.perf_counter()
        assert cli.main(loop + extra) == 0
        torch.cuda.synchronize()
        if rep > 0:                                     # the first pair warms up the contexts and cuDNN's choices
            times[name].append(time.perf_counter() - t0)
rec["generation_loop"] = {"images": 256, "batch": 64, "nfe": 20,
                          "fid_s": [round(t, 3) for t in times["fid"]], "fid_is_s": [round(t, 3) for t in times["fid_is"]],
                          "is_added_s": round(min(times["fid_is"]) - min(times["fid"]), 3)}
print(json.dumps(rec["generation_loop"]), flush=True)
shutil.rmtree(tmp, ignore_errors=True)
if len(sys.argv) > 1:
    os.makedirs(sys.argv[1], exist_ok=True)
    with open(os.path.join(sys.argv[1], "is_profile.json"), "w") as f:
        json.dump(rec, f, indent=1)
