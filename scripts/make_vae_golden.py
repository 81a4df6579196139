"""Record tests/golden/vae_decode_fingerprint.npz: fingerprints of the native VAE decode at latent 16 and 32 (128 and 256 pixel
images) on cuda:0, with the synthetic decoder weights of oracle/vae.py (seed 1) and seeded latents.

    python scripts/make_vae_golden.py [OUT.npz]

Per case it stores the SHA-256 of the fp32 `sample` bytes and of the fused uint8 image bytes, and a strided subsample of the fp32
sample (so that a mismatch can be located).  tests/test_gpu_vae512.py decodes the same latents and requires the same bytes: the
512-pixel decode must leave the smaller decodes bit-identical.  The decode plans split-K by the SM count, so the fingerprint
also records it (132 on an H100 SXM)."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from oracle import vae as ovae  # noqa: E402

# (latent side, batch, max_batch): the shapes of test_vae_decode_vs_oracle (an odd batch split across decode chunks)
CASES = [(16, 3, 2), (32, 2, 2)]
STRIDE = 61


def latents(side, B):
    g = torch.Generator().manual_seed(100 + side)
    return torch.randn(B, 4, side, side, generator=g) / 0.18215 * 0.2


def fingerprint(side, B, max_batch, dev):
    vae = lfm_b200.AutoencoderKL(max_batch=max_batch)
    vae.load_state_dict(ovae.synthetic_state_dict(ovae.VAEConfig(), 1), strict=True)
    vae = vae.to(dev).eval()
    z = latents(side, B).to(dev)
    out = vae.decode(z).sample.cpu().contiguous()
    u8 = vae.decode_to_uint8(z).cpu().contiguous()
    return {f"s{side}_f32_sha256": hashlib.sha256(out.numpy().tobytes()).hexdigest(),
            f"s{side}_u8_sha256": hashlib.sha256(u8.numpy().tobytes()).hexdigest(),
            f"s{side}_f32_sub": out.reshape(-1)[::STRIDE].numpy().copy()}


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "vae_decode_fingerprint.npz")
    dev = torch.device("cuda:0")
    rec = {"num_sms": np.int64(torch.cuda.get_device_properties(0).multi_processor_count),
           "device": torch.cuda.get_device_name(0), "stride": np.int64(STRIDE)}
    for side, B, mb in CASES:
        rec.update(fingerprint(side, B, mb, dev))
    np.savez_compressed(out, **rec)
    print({k: (v if isinstance(v, str) else getattr(v, "shape", v)) for k, v in rec.items()})


if __name__ == "__main__":
    main()
