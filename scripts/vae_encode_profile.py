"""Timing of the native VAE encode (lfm_b200.AutoencoderKL(with_encoder=True).encode, synthetic weights) on cuda:0: ms per
image, images/s, TFLOP/s and launches per encode, at batch 16 for 256-pixel images and batch 4 for 512-pixel images, next to
the card's name and power limit.
python scripts/vae_encode_profile.py [side:batch ...]      (default: 256:16 512:4)"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402

dev = torch.device("cuda:0")
cases = [tuple(int(v) for v in a.split(":")) for a in sys.argv[1:]] or [(256, 16), (512, 4)]
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True, timeout=30).stdout.strip()
print(json.dumps({"gpu": q or torch.cuda.get_device_name(0)}), flush=True)
for side, B in cases:
    vae = lfm_b200.AutoencoderKL(with_encoder=True, max_batch=B if side < 512 else 4 * B)
    vae.load_state_dict(lfm_b200.synthetic_vae_state_dict(vae, 1), strict=True)
    vae = vae.to(dev).eval()
    x = torch.rand(B, 3, side, side, device=dev) * 2 - 1
    for _ in range(2):
        dist = vae.encode(x).latent_dist
    torch.cuda.synchronize()
    reps = 10
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = vae._enc_native.launch_count()
    e0.record()
    for _ in range(reps):
        dist = vae.encode(x).latent_dist
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = vae.encode_flops_per_image(side)
    print(json.dumps({"vae_encode_side": side, "batch": B, "ms": round(ms, 3), "ms_per_image": round(ms / B, 3),
                      "images_per_s": round(B / ms * 1e3, 1), "tflop_per_image": round(fl / 1e12, 3),
                      "tflops": round(B * fl / ms / 1e9, 1), "encode_calls": -(-B // vae.decode_chunk(side // 8)),
                      "launches_per_encode": (vae._enc_native.launch_count() - l0) // reps,
                      "finite": bool(torch.isfinite(dist.mean).all() and torch.isfinite(dist.logvar).all())}), flush=True)
    del vae, dist
    torch.cuda.empty_cache()
