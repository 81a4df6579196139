"""Timing of semantic synthesis on cuda:0, next to the card's name and power limit.

1. The condition stage of a batch of 64 label maps at 256 x 256, for 19 (CelebAMask-HQ) and 182 (COCO) classes:
   SpatialRescaler.forward_labels (one kernel on the uint8 labels) against the reference's torch route,
   ``cond_stage_model(F.one_hot(seg, K).permute(0, 3, 1, 2).float())`` on the device.  CUDA events, best of several repeats.
2. One full batch of the readme's semantic preset (``--attn_resolution 16 8``, batch 64, Euler with 50 steps, synthetic
   weights), split into condition, sampling and decode.  Adaptive solvers on synthetic weights take a number of steps a trained
   model would not, so the timing uses Euler.

python scripts/semantic_profile.py"""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lfm_b200 import cli_semantic  # noqa: E402
from lfm_b200.downstream import SpatialRescaler, WrapperCondFlow, sample_from_model  # noqa: E402

torch.set_grad_enabled(False)
dev = torch.device("cuda:0")
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True, timeout=30).stdout.strip()
print(json.dumps({"gpu": q or torch.cuda.get_device_name(0)}), flush=True)


def best_ms(fn, reps=5, iters=10):
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


B, S = 64, 256
for K in (19, 182):
    m = SpatialRescaler(n_stages=3, in_channels=K, out_channels=4, multiplier=0.5)
    m.load_state_dict({"channel_mapper.weight": torch.randn(4, K, 1, 1, generator=torch.Generator().manual_seed(K)) / K ** 0.5})
    m = m.to(dev).eval()
    seg = torch.randint(0, K, (B, S, S), generator=torch.Generator().manual_seed(1)).to(torch.uint8).to(dev)
    seg_long = seg.long()
    native = best_ms(lambda: m.forward_labels(seg))
    onehot = best_ms(lambda: m(F.one_hot(seg_long, K).permute(0, 3, 1, 2).float()), reps=3, iters=3)
    diff = float((m.forward_labels(seg) - m(F.one_hot(seg_long, K).permute(0, 3, 1, 2).float())).abs().max())
    print(json.dumps({"condition_classes": K, "batch": B, "side": S, "forward_labels_ms": round(native, 4),
                      "torch_one_hot_ms": round(onehot, 3), "speedup": round(onehot / native, 1),
                      "label_bytes": B * S * S, "one_hot_int64_bytes": B * S * S * K * 8, "max_abs_diff": diff}), flush=True)
    del seg_long
    torch.cuda.empty_cache()

argv = ["--dataset", "celeba", "--attn_resolution", "16", "8", "--batch_size", str(B), "--method", "euler",
        "--step_size", "0.02", "--synthetic_init", "1", "--synthetic_vae", "2", "--device", "cuda:0"]
args = cli_semantic.parse_args(argv)
model, cond, vae = cli_semantic.load(args, dev)
seg = torch.randint(0, 19, (B, S, S), generator=torch.Generator().manual_seed(2)).to(torch.uint8).to(dev)
z_0 = torch.randn(B, 4, S // 8, S // 8, generator=torch.Generator().manual_seed(3)).to(dev)
stages = {}
for rep in range(3):                                         # the first repeat builds the contexts and graphs
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    c = cond.forward_labels(seg)
    ev[1].record()
    fake = sample_from_model(WrapperCondFlow(model, c), z_0, args)[-1]
    ev[2].record()
    img = (vae.decode(fake / args.scale_factor).sample + 1.0) / 2.0
    ev[3].record()
    torch.cuda.synchronize()
    if rep > 0:
        for name, a, b in (("condition", 0, 1), ("sampling", 1, 2), ("decode", 2, 3)):
            stages[name] = min(stages.get(name, float("inf")), ev[a].elapsed_time(ev[b]))
total = sum(stages.values())
print(json.dumps({"semantic_batch": B, "preset": "attn 16 8, Euler-50, synthetic weights",
                  **{k + "_ms": round(v, 3) for k, v in stages.items()}, "total_ms": round(total, 1),
                  "ms_per_image": round(total / B, 2), "finite": bool(torch.isfinite(img).all())}), flush=True)
