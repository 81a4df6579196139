"""Record tests/golden/dit_fingerprint.npz: fingerprints of the DiT forward (lfm_forward) on the mini_uncond, mini_cond and
mini_xl2 fixtures, of the uniform-row forward (0-d t, no labels) and a 4-step Euler run without labels on mini_uncond, and of
a 4-step Euler run with CFG on mini_cond, each in the bf16 and the FP8 mode, on cuda:0.

    python scripts/make_dit_golden.py [OUT.npz]

The weights are the fixtures' own (oracle.dit.synthetic_state_dict with their weight_seed), the inputs their stored latents,
times and labels.  Per case it stores the SHA-256 of the fp32 output bytes and a strided subsample (so that a mismatch can be
located).  tests/test_gpu_dit_fingerprint.py computes the same outputs and requires the same bytes: a change to the DiT's host
code that is meant to keep its numerics must keep them bit for bit.  The GEMM tile width follows the SM count, so the
fingerprint also records it (132 on an H100 SXM)."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lfm_b200  # noqa: E402
from oracle import dit as odit  # noqa: E402

STRIDE = 37
FIXTURES = ("mini_uncond", "mini_cond", "mini_xl2")


def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    g = {k: z[k] for k in z.files}
    cfg = odit.DiTConfig(img_resolution=int(g["cfg_img_resolution"]), patch_size=int(g["cfg_patch_size"]),
                         in_channels=int(g["cfg_in_channels"]), hidden_size=int(g["cfg_hidden_size"]),
                         depth=int(g["cfg_depth"]), num_heads=int(g["cfg_num_heads"]),
                         label_dropout=float(g["cfg_label_dropout"]), num_classes=int(g["cfg_num_classes"]))
    return g, cfg


def _net(g, cfg, fp8, dev):
    net = lfm_b200.DiT(img_resolution=cfg.img_resolution, patch_size=cfg.patch_size, in_channels=cfg.in_channels,
                       hidden_size=cfg.hidden_size, depth=cfg.depth, num_heads=cfg.num_heads,
                       label_dropout=cfg.label_dropout, num_classes=cfg.num_classes, fp8=fp8)
    net.load_state_dict(odit.synthetic_state_dict(cfg, int(g["weight_seed"])), strict=True)
    return net.to(dev).eval()


def outputs(dev):
    """name -> fp32 CPU tensor: per mode, one forward on each fixture ([B] t, labels), the uniform-row forward and Euler-4
    without labels on mini_uncond, and Euler-4 with CFG 1.5 on mini_cond."""
    res = {}
    for mode in ("bf16", "fp8"):
        for name in FIXTURES:
            g, cfg = _fixture(name)
            net = _net(g, cfg, mode == "fp8", dev)
            t, x, y = (torch.from_numpy(np.asarray(g[k])).to(dev) for k in ("t_vec", "x", "y"))
            res[f"{mode}_{name}_forward"] = net(t, x, y).cpu()
            if name == "mini_uncond":
                # a 0-d t without labels: one conditioning row, read by every sample with stride 0
                res[f"{mode}_{name}_forward_uniform"] = net(torch.tensor(float(g["t_scalar"]), device=dev), x).cpu()
                out = lfm_b200.karras_sample(net, x, 5, clip_denoised=False, model_kwargs={}, sigma_min=1e-5, sigma_max=1.0,
                                             sampler="euler")
                assert net.last_stats["nfe"] == 4
                res[f"{mode}_{name}_euler4"] = out.cpu()
            if name == "mini_cond":
                mk = dict(y=torch.from_numpy(np.asarray(g["y_cfg"])).to(dev), cfg_scale=1.5)
                out = lfm_b200.karras_sample(net, torch.cat([x, x]), 5, clip_denoised=False, model_kwargs=mk, sigma_min=1e-5,
                                             sigma_max=1.0, sampler="euler")
                assert net.last_stats["nfe"] == 4
                res[f"{mode}_{name}_euler4_cfg"] = out.cpu()
    return res


def fingerprint(dev):
    rec = {}
    for k, v in outputs(dev).items():
        v = v.float().contiguous()
        rec[k + "_sha256"] = hashlib.sha256(v.numpy().tobytes()).hexdigest()
        rec[k + "_sub"] = v.reshape(-1)[::STRIDE].numpy().copy()
    return rec


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "dit_fingerprint.npz")
    dev = torch.device("cuda:0")
    rec = {"num_sms": np.int64(torch.cuda.get_device_properties(0).multi_processor_count),
           "device": torch.cuda.get_device_name(0), "stride": np.int64(STRIDE)}
    rec.update(fingerprint(dev))
    np.savez_compressed(out, **rec)
    print({k: (v if isinstance(v, str) else getattr(v, "shape", v)) for k, v in rec.items()})


if __name__ == "__main__":
    main()
