"""H100-native decoder of the Stable-Diffusion ``AutoencoderKL`` - the VAE decode step of the sampling path
(``first_stage_model.decode(fake_sample / args.scale_factor).sample``, test_flow_latent.py:131,193;
test_flow_latent_ddp.py:57,110).

``diffusers`` is a third-party dependency of the reference that is absent from this image, so this class mirrors the
part of its interface the reference uses: ``AutoencoderKL.from_pretrained(dir)`` (a LOCAL diffusers-format directory:
``config.json`` + ``diffusion_pytorch_model.safetensors`` / ``.bin``; there is no network here), ``.to(device)``,
``.decode(z).sample``.  Parameters live in an ``nn.Module`` tree with the diffusers ``state_dict`` keys of the decoder
(``decoder.*``, ``post_quant_conv.*``; a full checkpoint's ``encoder.*`` / ``quant_conv.*`` entries are ignored, legacy
attention names are renamed as diffusers does); the compute is liblfm_b200.so (``lfm_create_vae`` / ``lfm_decode``:
wgmma implicit-GEMM convolutions, fused GroupNorm + SiLU, tensor-core attention GEMMs).  ``decode_to_uint8`` also
fuses the generation loop's post-processing (test_flow_latent_ddp.py:131-135).  No PyTorch forward, no fallback.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import types

import torch
import torch.nn as nn

from . import _lib
from .network import _Holder, _NativeNet

LEGACY_ATTN = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def _resnet(cin, cout):
    b = _Holder()
    b.norm1 = nn.GroupNorm(32, cin, eps=1e-6)
    b.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
    b.norm2 = nn.GroupNorm(32, cout, eps=1e-6)
    b.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
    if cin != cout:
        b.conv_shortcut = nn.Conv2d(cin, cout, 1)
    return b


class _List(nn.Module):
    def __init__(self, mods):
        super().__init__()
        for i, m in enumerate(mods):
            self.add_module(str(i), m)

    def __getitem__(self, i):
        return getattr(self, str(i))


class AutoencoderKL(_NativeNet):
    """Decoder-only mirror of ``diffusers.AutoencoderKL`` (defaults = the stabilityai/sd-vae-ft-mse config)."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, norm_num_groups=32, scaling_factor=0.18215, max_batch=16, **unused):
        super().__init__()
        self.block_out_channels = tuple(int(c) for c in block_out_channels)
        self.layers_per_block, self.latent_channels, self.out_channels = int(layers_per_block), int(latent_channels), int(out_channels)
        self.norm_num_groups = int(norm_num_groups)
        self.config = types.SimpleNamespace(scaling_factor=scaling_factor, block_out_channels=self.block_out_channels,
                                            layers_per_block=self.layers_per_block, latent_channels=self.latent_channels)
        self.max_batch_hint = max_batch
        rev = self.block_out_channels[::-1]
        dec = _Holder()
        dec.conv_in = nn.Conv2d(latent_channels, rev[0], 3, padding=1)
        ups, ch = [], rev[0]
        for i, out in enumerate(rev):
            blk = _Holder()
            res = []
            for _ in range(self.layers_per_block + 1):
                res.append(_resnet(ch, out))
                ch = out
            blk.resnets = _List(res)
            if i != len(rev) - 1:
                up = _Holder()
                up.conv = nn.Conv2d(ch, ch, 3, padding=1)
                blk.upsamplers = _List([up])
            ups.append(blk)
        dec.up_blocks = _List(ups)
        mid = _Holder()
        att = _Holder()
        att.group_norm = nn.GroupNorm(32, rev[0], eps=1e-6)
        att.to_q = nn.Linear(rev[0], rev[0])
        att.to_k = nn.Linear(rev[0], rev[0])
        att.to_v = nn.Linear(rev[0], rev[0])
        att.to_out = _List([nn.Linear(rev[0], rev[0])])
        mid.attentions = _List([att])
        mid.resnets = _List([_resnet(rev[0], rev[0]), _resnet(rev[0], rev[0])])
        dec.mid_block = mid
        dec.conv_norm_out = nn.GroupNorm(32, ch, eps=1e-6)
        dec.conv_out = nn.Conv2d(ch, out_channels, 3, padding=1)
        self.decoder = dec
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.requires_grad_(False)
        self._init_native()
        self._latent_size = None

    # -- loading ------------------------------------------------------------------------------------------------------
    @staticmethod
    def decoder_state_dict(sd):
        """The entries of a (possibly full, possibly legacy-named) AutoencoderKL checkpoint this module holds."""
        out = {}
        for k, v in sd.items():
            if not (k.startswith("decoder.") or k.startswith("post_quant_conv.")):
                continue
            parts = k.split(".")
            if "attentions" in parts and len(parts) >= 2 and parts[-2] in LEGACY_ATTN:
                parts[-2] = LEGACY_ATTN[parts[-2]]
                if v.dim() == 4:          # very old checkpoints store the projections as 1x1 convolutions
                    v = v[:, :, 0, 0]
            out[".".join(parts)] = v
        return out

    def load_state_dict(self, state_dict, strict=True, **kw):
        return super().load_state_dict(self.decoder_state_dict(state_dict), strict=strict, **kw)

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **kwargs):
        """``AutoencoderKL.from_pretrained`` for a LOCAL diffusers directory (no hub access in this environment)."""
        root = os.path.join(path, subfolder) if subfolder else path
        cfg_path = os.path.join(root, "config.json")
        if not os.path.isfile(cfg_path):
            raise FileNotFoundError(
                f"{root!r} is not a local diffusers AutoencoderKL directory (config.json missing); downloading "
                f"'{path}' from the hub is not possible offline - pass a local copy, or use synthetic weights")
        with open(cfg_path) as f:
            cfg = json.load(f)
        keep = ("in_channels", "out_channels", "block_out_channels", "layers_per_block", "latent_channels", "norm_num_groups",
                "scaling_factor")
        vae = cls(**{k: cfg[k] for k in keep if k in cfg}, **kwargs)
        st = os.path.join(root, "diffusion_pytorch_model.safetensors")
        if os.path.isfile(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(root, "diffusion_pytorch_model.bin"), map_location="cpu")
        vae.load_state_dict(sd, strict=True)
        return vae.eval()

    # -- native context -------------------------------------------------------------------------------------------------
    def _version(self):
        return (self._latent_size,) + super()._version()

    def _create_ctx(self, lib, dev_index):
        boc = self.block_out_channels
        d = _lib.VaeDesc(self._latent_size, self.latent_channels, self.out_channels, len(boc), (C.c_int32 * 8)(*boc),
                         self.layers_per_block, self.norm_num_groups)
        ctx = C.c_void_p()
        _lib.check(lib.lfm_create_vae(C.byref(d), dev_index, C.byref(ctx)))
        return ctx

    def _decode_native(self, z, want_f32, want_u8):
        if not z.is_cuda:
            raise RuntimeError("lfm_b200: z must be a CUDA tensor (no CPU path)")
        z = z.to(torch.float32).contiguous()
        B, Cc, h, w = z.shape
        if Cc != self.latent_channels or h != w:
            raise ValueError(f"expected square latents [B, {self.latent_channels}, s, s], got {tuple(z.shape)}")
        if self._latent_size != h:
            self._latent_size = h
            self._dirty = True              # another latent size = another native context
        up = 2 ** (len(self.block_out_channels) - 1)
        out = torch.empty(B, self.out_channels, h * up, w * up, device=z.device) if want_f32 else None
        u8 = torch.empty(B, h * up, w * up, self.out_channels, device=z.device, dtype=torch.uint8) if want_u8 else None
        chunk = max(1, int(self.max_batch_hint or 16))
        ctx = self.native(min(B, chunk), z.device)
        lib = _lib.load()
        for i in range(0, B, chunk):
            n = min(chunk, B - i)
            _lib.check(lib.lfm_decode(ctx, z[i:i + n].data_ptr(), n, out[i:i + n].data_ptr() if want_f32 else None,
                                      u8[i:i + n].data_ptr() if want_u8 else None, self._stream(z.device)), ctx)
        return out, u8

    # -- first_stage_model.decode(z).sample  (test_flow_latent.py:193) --------------------------------------------------
    def decode(self, z, return_dict=True, **kwargs):
        sample, _ = self._decode_native(z, True, False)
        return types.SimpleNamespace(sample=sample) if return_dict else (sample,)

    def decode_to_uint8(self, z):
        """decode + ``(clamp((x + 1) / 2, 0, 1) * 255).permute(0, 2, 3, 1).to(uint8)`` (test_flow_latent_ddp.py:131-135)
        in one pass: [B, 4, s, s] latents -> [B, 8s, 8s, 3] uint8 on the device."""
        return self._decode_native(z, False, True)[1]

    def forward(self, *a, **k):
        raise NotImplementedError("only the decoder of the AutoencoderKL is on the sampling path: use .decode(z)")

    def decode_flops_per_image(self, latent_side: int = 32) -> float:
        """Algorithmic FLOPs (2 x MAC) of one decode: the convolutions, the four attention projections and the two
        attention GEMMs (the figure bench.py's decode roofline uses)."""
        rev = self.block_out_channels[::-1]
        L, c0 = self.latent_channels, rev[0]
        side = latent_side
        px = side * side
        fl = 2.0 * px * (L * L + 9 * L * c0)
        fl += 2 * (2.0 * px * 9 * 2 * c0 * c0) + 2.0 * px * 4 * c0 * c0 + 4.0 * px * px * c0        # mid block
        ch = c0
        for i, out in enumerate(rev):
            px = side * side
            for _ in range(self.layers_per_block + 1):
                fl += 2.0 * px * 9 * (ch * out + out * out) + (2.0 * px * ch * out if ch != out else 0.0)
                ch = out
            if i != len(rev) - 1:
                side *= 2
                fl += 2.0 * side * side * 9 * ch * ch
        fl += 2.0 * side * side * 9 * ch * self.out_channels
        return fl


def synthetic_vae_state_dict(vae: AutoencoderKL, seed: int = 1):
    """Seeded non-degenerate decoder weights (the real sd-vae-ft-mse file is a network download): conv / linear
    U(-a, a) with a = 1/sqrt(fan_in); GroupNorm weight 1 + 0.1 N, bias 0.1 N; biases 0.02 N.  Every tensor has its own
    generator seeded from (seed, crc32(key)), so the result does not depend on the key order; same recipe as
    oracle.vae.synthetic_state_dict (tests/test_host_logic.py checks they agree)."""
    import zlib
    sd = {}
    for k, v in vae.state_dict().items():
        shp = tuple(v.shape)
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(k.encode()))
        leaf = k.rsplit(".", 2)[-2]
        if "norm" in leaf:
            sd[k] = (1.0 + 0.1 * torch.randn(shp, generator=g)) if k.endswith("weight") else 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            sd[k] = 0.02 * torch.randn(shp, generator=g)
        else:
            fan_in = int(math.prod(shp[1:]))
            sd[k] = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
    return sd
