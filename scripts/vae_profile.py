"""Timing of the native VAE decode (lfm_b200.AutoencoderKL, synthetic weights) on cuda:0: ms per batch, images/s, TFLOP/s,
launches per decode, and the device memory the native context takes per image of its batch.
python scripts/vae_profile.py [--latent {32,64}] [batch ...]
(latent 32: 256 x 256 images, default batches 1 16 64; latent 64: 512 x 512 images, default batches 1 4)"""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402

p = argparse.ArgumentParser()
p.add_argument("--latent", type=int, default=32, choices=[32, 64])
p.add_argument("batches", type=int, nargs="*")
args = p.parse_args()
dev = torch.device("cuda:0")
S = args.latent


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0)
    return q


def make_vae(max_batch):
    vae = lfm_b200.AutoencoderKL(max_batch=max_batch)
    vae.load_state_dict(lfm_b200.synthetic_vae_state_dict(vae, 1), strict=True)
    return vae.to(dev).eval()


def context_bytes(max_batch):
    """Device memory taken by the native context (weights + workspace) sized for vae.decode_chunk(S) images."""
    vae = make_vae(max_batch)
    z = torch.randn(1, 4, S, S, device=dev)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    vae.decode_to_uint8(z)
    torch.cuda.synchronize()
    used = free0 - torch.cuda.mem_get_info(0)[0]
    rows = vae.decode_chunk(S)
    del vae
    gc.collect()
    torch.cuda.synchronize()
    return rows, used


print(json.dumps({"gpu": gpu_info(), "latent": S, "image_side": 8 * S}), flush=True)
(r1, b1), (r4, b4) = context_bytes(1), context_bytes(4 if S < 64 else 16)
print(json.dumps({"context_rows": [r1, r4], "context_MB": [round(b1 / 2**20), round(b4 / 2**20)],
                  "workspace_MB_per_image": round((b4 - b1) / (r4 - r1) / 2**20, 1)}), flush=True)

vae = make_vae(16)
fl = vae.decode_flops_per_image(S)
for B in args.batches or ([1, 16, 64] if S == 32 else [1, 4]):
    z = torch.randn(B, 4, S, S, device=dev) * 1.1
    for _ in range(2):
        u8 = vae.decode_to_uint8(z)
    torch.cuda.synchronize()
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = vae.launch_count()
    e0.record()
    for _ in range(reps):
        u8 = vae.decode_to_uint8(z)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    chunks = -(-B // vae.decode_chunk(S))
    print(json.dumps({"vae_decode_batch": B, "latent": S, "ms": round(ms, 3), "ms_per_image": round(ms / B, 3),
                      "images_per_s": round(B / ms * 1e3, 1), "tflop_per_image": round(fl / 1e12, 3),
                      "tflops": round(B * fl / ms / 1e9, 1), "decode_calls": chunks,
                      "launches_per_decode": (vae.launch_count() - l0) // reps,
                      "finite": bool(torch.isfinite(vae.decode(z[:1]).sample).all())}), flush=True)
