"""DiT-L/2 forward, batch 64 (the headline workload's network evaluation) - used under ncu and for timing.
usage: dit_profile.py [batch] [iters] [model_type] [latent side] [--kernel-table DIR]
  --kernel-table DIR: also record `iters` forwards under torch.profiler (CUDA activities) and write the per-kernel table -
  kernel, launches per NFE, microseconds per NFE, share of the NFE's kernel time - to DIR/kernel_table.{md,json}, with the
  card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from lfm_b200.synthetic import synthetic_state_dict  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("batch", type=int, nargs="?", default=64)
ap.add_argument("iters", type=int, nargs="?", default=20)
ap.add_argument("model_type", nargs="?", default="DiT-L/2")
ap.add_argument("side", type=int, nargs="?", default=32)
ap.add_argument("--kernel-table", metavar="DIR", default=None)
args = ap.parse_args()
B, iters, mt, S = args.batch, args.iters, args.model_type, args.side
dev = torch.device("cuda:0")
with torch.device("meta"):
    net = lfm_b200.DiT_models[mt](img_resolution=S, in_channels=4, label_dropout=0.0, num_classes=1)
# algorithmic FLOPs per sample per evaluation (SURVEY.md 8(d)): 161,386,856,448 for DiT-L/2, 46,003,912,704 for DiT-B/2
L_, D_, P_ = net.depth, net.hidden_size, net.patch_size ** 2 * net.in_channels
T_ = (net.img_resolution // net.patch_size) ** 2
FLOPS = L_ * (24 * T_ * D_ * D_ + 4 * T_ * T_ * D_ + 12 * D_ * D_) + 2 * T_ * P_ * D_ + 2 * (256 * D_ + D_ * D_) + 4 * D_ * D_ + 2 * T_ * D_ * P_
sd = synthetic_state_dict(net, 1)
net = net.to_empty(device="cpu")
net.load_state_dict(sd, strict=True)
net = net.to(dev)
x = torch.randn(B, 4, S, S, device=dev)
t = torch.tensor(0.5, device=dev)
for _ in range(3):
    net(t, x)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(iters):
    v = net(t, x)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
print(f"{mt} ({S}x{S} latents) forward B={B}: {ms:.3f} ms/NFE, {B * FLOPS / ms / 1e9:.1f} TFLOP/s, launches/NFE {net.launch_count() // (iters + 3)}")

if args.kernel_table:
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            net(t, x)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.name.startswith("Memcpy") or ev.name.startswith("Memset"):
            continue
        name = ev.name.removeprefix("void ").split("(")[0].removeprefix("lfm::")
        r = rows.setdefault(name, [0, 0.0])
        r[0] += 1
        r[1] += ev.device_time
    total = sum(us for _, us in rows.values())
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    table = [{"kernel": k, "launches_per_nfe": n / iters, "us_per_nfe": round(us / iters, 1), "share": round(us / total, 4)}
             for k, (n, us) in sorted(rows.items(), key=lambda kv: -kv[1][1])]
    os.makedirs(args.kernel_table, exist_ok=True)
    with open(os.path.join(args.kernel_table, "kernel_table.json"), "w") as f:
        json.dump({"gpu": gpu, "model": mt, "batch": B, "side": S, "nfe_ms_unprofiled": round(ms, 3),
                   "kernel_us_per_nfe": round(total / iters, 1), "kernels": table}, f, indent=1)
    lines = [f"{mt} forward, batch {B}, {S}x{S} latents, {iters} NFEs under torch.profiler; GPU: {gpu}",
             f"unprofiled {ms:.3f} ms/NFE; kernel time {total / iters / 1e3:.3f} ms/NFE", "",
             "| kernel | launches / NFE | us / NFE | share |", "|---|---|---|---|"]
    lines += [f"| `{r['kernel']}` | {r['launches_per_nfe']:g} | {r['us_per_nfe']:.1f} | {100 * r['share']:.1f}% |" for r in table]
    with open(os.path.join(args.kernel_table, "kernel_table.md"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))
