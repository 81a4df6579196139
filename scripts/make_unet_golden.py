"""Record tests/golden/unet_fingerprint.npz: fingerprints of a 4-channel UNetModel forward, of a celeb512-preset dopri5
trajectory, of the class-conditional unet_mini_cond forward, and of the DhariwalUNet (EDM) forwards on the edm_mini and
edm_mini_cond fixtures (with and without labels, and forward_with_cfg) with a CFG Euler-4 run on edm_mini_cond, on cuda:0.
The celeb networks have seeded synthetic weights and latents; the fixtures' networks have their own weights and inputs.

    python scripts/make_unet_golden.py [OUT.npz]

Per case it stores the SHA-256 of the fp32 output bytes and a strided subsample (so that a mismatch can be located).
tests/test_gpu_downstream.py computes the same outputs and requires the same bytes: a change to the UNet program's host
code that is meant to keep its numerics must keep them bit for bit.  The network plans split-K by the SM count, so the
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
from oracle import edm as oedm  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from tests.test_oracle_edm import edm_cfg_from_golden  # noqa: E402
from tests.test_oracle_unet import unet_cfg_from_golden  # noqa: E402

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


def _fixture(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    return {k: z[k] for k in z.files}


def _fixture_net(name, dev):
    """The fixture's network with its own weights (unet_* -> UNetModel, edm_* -> DhariwalUNet) and the fixture."""
    g = _fixture(name)
    if name.startswith("unet_"):
        c = unet_cfg_from_golden(g)
        net = lfm_b200.UNetModel(image_size=c.image_size, in_channels=4, model_channels=c.model_channels, out_channels=4,
                                 num_res_blocks=c.num_res_blocks, attention_resolutions=c.attention_resolutions,
                                 channel_mult=c.channel_mult, num_classes=c.num_classes, num_heads=c.num_heads,
                                 num_head_channels=c.num_head_channels, use_scale_shift_norm=True)
        sd = ounet.synthetic_state_dict(c, int(g["weight_seed"]))
    else:
        c = edm_cfg_from_golden(g)
        net = lfm_b200.DhariwalUNet(img_resolution=c.img_resolution, in_channels=4, out_channels=4, label_dim=c.label_dim,
                                    model_channels=c.model_channels, channel_mult=c.channel_mult, num_blocks=c.num_blocks,
                                    attn_resolutions=c.attn_resolutions, dropout=0.0)
        sd = oedm.synthetic_state_dict(c, int(g["weight_seed"]))
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval(), {k: torch.from_numpy(np.asarray(v)).to(dev) for k, v in g.items()}


def outputs(dev):
    """name -> fp32 CPU tensor: one celeb256 forward (batch 3), a celeb512 dopri5 trajectory (batch 2, 1e-3), the forward of
    unet_mini_cond ([B] t, labels), of edm_mini ([B] t) and of edm_mini_cond ([B] t with and without labels, and
    forward_with_cfg 1.5), and Euler-4 with CFG 1.5 on edm_mini_cond."""
    g = torch.Generator().manual_seed(77)
    net = _net(32, (1, 2, 2, 2), 4, dev)
    x = torch.randn(3, 4, 32, 32, generator=g)
    res = {"celeb256_forward": net(torch.tensor([0.9, 0.5, 0.1], device=dev), x.to(dev)).cpu()}
    net = _net(64, (1, 2, 2, 2, 4), 2, dev)
    x = torch.randn(2, 4, 64, 64, generator=g)
    args = types.SimpleNamespace(method="dopri5", atol=1e-3, rtol=1e-3, cfg_scale=1.0, compute_nfe=False)
    res["celeb512_dopri5"] = lfm_b200.sample_from_model(net, x.to(dev), {}, args)[-1].cpu()
    net, g = _fixture_net("unet_mini_cond", dev)
    res["unet_mini_cond_forward"] = net(g["t_vec"], g["x"], g["y"]).cpu()
    net, g = _fixture_net("edm_mini", dev)
    res["edm_mini_forward"] = net(g["t_vec"], g["x"]).cpu()
    net, g = _fixture_net("edm_mini_cond", dev)
    x2 = torch.cat([g["x"], g["x"]])
    res["edm_mini_cond_forward"] = net(g["t_vec"], g["x"], g["y"]).cpu()
    res["edm_mini_cond_forward_nolabel"] = net(g["t_vec"], g["x"]).cpu()
    res["edm_mini_cond_forward_cfg"] = net.forward_with_cfg(g["t_cfg"], x2, g["y_cfg"], cfg_scale=1.5).cpu()
    out = lfm_b200.karras_sample(net, x2, 5, clip_denoised=False, model_kwargs=dict(y=g["y_cfg"], cfg_scale=1.5), sigma_min=1e-5,
                                 sigma_max=1.0, sampler="euler")
    assert net.last_stats["nfe"] == 4
    res["edm_mini_cond_euler4_cfg"] = out.cpu()
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
