"""Record tests/golden/unet_fingerprint.npz: fingerprints of a 4-channel UNetModel forward and of a celeb512-preset dopri5
trajectory on cuda:0, with seeded synthetic weights and latents.

    python scripts/make_unet_golden.py [OUT.npz]

Per case it stores the SHA-256 of the fp32 output bytes and a strided subsample (so that a mismatch can be located).
tests/test_gpu_downstream.py computes the same outputs and requires the same bytes: generalising conv_in to concatenated
conditions must leave the unconditioned networks bit-identical.  The network plans split-K by the SM count, so the
fingerprint also records it (132 on an H100 SXM)."""
import hashlib
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from lfm_b200.synthetic import synthetic_unet_state_dict  # noqa: E402

STRIDE = 37


def _net(image_size, channel_mult, max_batch, dev):
    with torch.device("meta"):
        net = lfm_b200.UNetModel(image_size=image_size, in_channels=4, model_channels=256, out_channels=4, num_res_blocks=2,
                                 attention_resolutions=(16, 8), channel_mult=channel_mult, num_heads=4,
                                 use_scale_shift_norm=True, max_batch=max_batch)
    sd = synthetic_unet_state_dict(net, 1)
    net = net.to_empty(device="cpu")
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval()


def outputs(dev):
    """name -> fp32 CPU tensor: one celeb256 forward (batch 3) and a celeb512 dopri5 trajectory (batch 2, 1e-3)."""
    g = torch.Generator().manual_seed(77)
    net = _net(32, (1, 2, 2, 2), 4, dev)
    x = torch.randn(3, 4, 32, 32, generator=g)
    res = {"celeb256_forward": net(torch.tensor([0.9, 0.5, 0.1], device=dev), x.to(dev)).cpu()}
    net = _net(64, (1, 2, 2, 2, 4), 2, dev)
    x = torch.randn(2, 4, 64, 64, generator=g)
    args = types.SimpleNamespace(method="dopri5", atol=1e-3, rtol=1e-3, cfg_scale=1.0, compute_nfe=False)
    res["celeb512_dopri5"] = lfm_b200.sample_from_model(net, x.to(dev), {}, args)[-1].cpu()
    return res


def fingerprint(dev):
    rec = {}
    for k, v in outputs(dev).items():
        v = v.contiguous()
        rec[k + "_sha256"] = hashlib.sha256(v.numpy().tobytes()).hexdigest()
        rec[k + "_sub"] = v.reshape(-1)[::STRIDE].numpy().copy()
    return rec


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "unet_fingerprint.npz")
    dev = torch.device("cuda:0")
    rec = {"num_sms": np.int64(torch.cuda.get_device_properties(0).multi_processor_count),
           "device": torch.cuda.get_device_name(0), "stride": np.int64(STRIDE)}
    rec.update(fingerprint(dev))
    np.savez_compressed(out, **rec)
    print({k: (v if isinstance(v, str) else getattr(v, "shape", v)) for k, v in rec.items()})


if __name__ == "__main__":
    main()
