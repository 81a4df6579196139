"""Write the concat-conditioned UNetModel and SpatialRescaler fixtures (tests/golden/unet_inpaint_mini.npz,
unet_semantic_mini.npz, spatial_rescaler.npz) from the UNMODIFIED reference modules.

Run:  python scripts/make_cond_goldens.py      (needs the reference checkout, LFM_REFERENCE; not the GPU machine)

The downstream tasks (downstream_tasks/test_flow_latent_inpainting.py, test_flow_latent_semantic_syn.py) wrap the ADM
UNetModel in WrapperCondFlow: v = model(t, cat([z, cond], 1)), 9 input channels for inpainting (latent + mask), 8 for
semantic synthesis.  Each fixture stores z, cond, t, one network evaluation and a torchdiffeq-style Euler trajectory of
the wrapped reference module; the weights are oracle.unet.synthetic_state_dict(cfg, seed), loaded with strict=True.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("LFM_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "timm_shim"))
sys.path.insert(0, REF)

from oracle import solvers as osol  # noqa: E402
from oracle import unet as ounet  # noqa: E402

CASES = {
    # name: (UNetConfig kwargs, weight seed, batch, euler step size)
    "unet_inpaint_mini": (dict(image_size=16, in_channels=9, model_channels=128, out_channels=4, num_res_blocks=1,
                               attention_resolutions=(2, 4), channel_mult=(1, 2, 2), num_heads=2, num_head_channels=-1,
                               num_classes=None), 41, 2, 0.25),
    "unet_semantic_mini": (dict(image_size=32, in_channels=8, model_channels=128, out_channels=4, num_res_blocks=1,
                                attention_resolutions=(4, 8), channel_mult=(1, 2, 3, 4), num_heads=4, num_head_channels=-1,
                                num_classes=None), 42, 2, 0.25),
}


def make_unet(g):
    from models.guided_diffusion.unet import UNetModel

    for name, (kw, seed, B, h) in CASES.items():
        cfg = ounet.UNetConfig(**kw)
        net = UNetModel(image_size=kw["image_size"], in_channels=kw["in_channels"], model_channels=kw["model_channels"],
                        out_channels=kw["out_channels"], num_res_blocks=kw["num_res_blocks"],
                        attention_resolutions=kw["attention_resolutions"], dropout=0.0, channel_mult=kw["channel_mult"],
                        conv_resample=True, dims=2, num_classes=None, use_checkpoint=False, use_fp16=False,
                        num_heads=kw["num_heads"], num_head_channels=kw["num_head_channels"], num_heads_upsample=-1,
                        use_scale_shift_norm=True, resblock_updown=False, use_new_attention_order=False)
        net.load_state_dict(ounet.synthetic_state_dict(cfg, seed), strict=True)
        net.eval()
        s = kw["image_size"]
        z = torch.randn(B, 4, s, s, generator=g)
        cond = torch.randn(B, kw["in_channels"] - 4, s, s, generator=g)
        tv = torch.tensor([0.8, 0.35][:B])
        # WrapperCondFlow.forward; a 0-d t is expanded to the batch here as unet.py:629-630 does (there on "cuda")
        f = lambda t, x: net(t * torch.ones(x.shape[0]) if t.dim() == 0 else t, torch.cat([x, cond], 1))  # noqa: E731
        out = {"z": z, "cond": cond, "t_vec": tv, "v": f(tv, z), "weight_seed": np.int64(seed), "euler_step": np.float64(h)}
        out["euler"] = osol.tdq_euler(f, z, h)[0]
        for k, v in kw.items():
            if v is not None and not isinstance(v, tuple):
                out["cfg_" + k] = np.float64(v)
        out["cfg_attention_resolutions"] = np.array(kw["attention_resolutions"], dtype=np.int64)
        out["cfg_channel_mult"] = np.array(kw["channel_mult"], dtype=np.int64)
        np.savez_compressed(os.path.join(OUT, name + ".npz"),
                            **{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in out.items()})
        print("wrote", name, "absmean(v)=%.4f" % float(out["v"].abs().mean()))


def make_spatial_rescaler(g):
    from models.encoder import SpatialRescaler

    m = SpatialRescaler(n_stages=3, in_channels=19, out_channels=4, multiplier=0.5)
    w = torch.randn(4, 19, 1, 1, generator=g) / 19 ** 0.5
    m.load_state_dict({"channel_mapper.weight": w}, strict=True)
    seg = torch.randint(0, 19, (2, 256, 256), generator=g)
    x = torch.nn.functional.one_hot(seg, 19).permute(0, 3, 1, 2).float()
    np.savez_compressed(os.path.join(OUT, "spatial_rescaler.npz"), seg=seg.numpy().astype(np.uint8), weight=w.numpy(),
                        out=m(x).numpy())
    print("wrote spatial_rescaler")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    make_unet(torch.Generator().manual_seed(9753))
    make_spatial_rescaler(torch.Generator().manual_seed(8642))
