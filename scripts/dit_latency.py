"""Small-batch latency of the sampling call (the reference's --measure_time protocol, test_flow_latent.py:223-246: CUDA events
around the solver call, batch 1): ms per network evaluation of DiT-L/2 inside graph-replayed Euler steps, batch 1 ... 16.
usage: dit_latency.py [model_type] [nfe] [reps] [batches, comma separated]"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from lfm_b200.synthetic import synthetic_state_dict  # noqa: E402

mt = sys.argv[1] if len(sys.argv) > 1 else "DiT-L/2"
nfe = int(sys.argv[2]) if len(sys.argv) > 2 else 20
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
batches = [int(b) for b in (sys.argv[4] if len(sys.argv) > 4 else "1,2,4,8,16").split(",")]
dev = torch.device("cuda:0")
with torch.device("meta"):
    net = lfm_b200.DiT_models[mt](img_resolution=32, in_channels=4, label_dropout=0.0, num_classes=1, max_batch=max(batches))
L_, D_, P_ = net.depth, net.hidden_size, net.patch_size ** 2 * net.in_channels
T_ = (net.img_resolution // net.patch_size) ** 2
FLOPS = L_ * (24 * T_ * D_ * D_ + 4 * T_ * T_ * D_ + 12 * D_ * D_) + 2 * T_ * P_ * D_ + 2 * (256 * D_ + D_ * D_) + 4 * D_ * D_ + 2 * T_ * D_ * P_
sd = synthetic_state_dict(net, 1)
net = net.to_empty(device="cpu")
net.load_state_dict(sd, strict=True)
net = net.to(dev).eval()
args = types.SimpleNamespace(method="euler", step_size=1.0 / nfe, cfg_scale=1.0)
for B in batches:
    x = torch.randn(B, 4, 32, 32, device=dev)
    for _ in range(2):
        lfm_b200.sample_from_model(net, x, {}, args)
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lfm_b200.sample_from_model(net, x, {}, args)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    per = ms / net.last_stats["nfe"]
    tf = f", {B * FLOPS / per / 1e9:.0f} TFLOP/s" if FLOPS else ""
    print(f"{mt} Euler-{nfe} batch {B}: {ms:.2f} ms per call, {per:.3f} ms/NFE, {B / ms * 1e3:.1f} img/s{tf}", flush=True)
