"""H100-native decoder of the Stable-Diffusion ``AutoencoderKL`` - the VAE decode step of the sampling path
(``first_stage_model.decode(fake_sample / args.scale_factor).sample``, test_flow_latent.py:131,193;
test_flow_latent_ddp.py:57,110) - and, with ``with_encoder=True``, its encoder (the inpainting loop's
``first_stage_model.encode(masked_image).latent_dist.sample()``, downstream_tasks/test_flow_latent_inpainting.py:147).

``diffusers`` is a third-party dependency of the reference that is absent from this image, so this class mirrors the
part of its interface the reference uses: ``AutoencoderKL.from_pretrained(dir)`` (a LOCAL diffusers-format directory:
``config.json`` + ``diffusion_pytorch_model.safetensors`` / ``.bin``; there is no network here), ``.to(device)``,
``.decode(z).sample``, ``.encode(x).latent_dist``.  Parameters live in an ``nn.Module`` tree with the diffusers
``state_dict`` keys of the decoder (``decoder.*``, ``post_quant_conv.*``; by default a full checkpoint's ``encoder.*`` /
``quant_conv.*`` entries are ignored) and, with ``with_encoder=True``, of the encoder too; legacy attention names are
renamed as diffusers does.  The compute is liblfm_b200.so: ``lfm_create_vae`` / ``lfm_decode`` and
``lfm_create_vae_encoder`` / ``lfm_encode``, two native contexts that each hold their own half of the weights
(wgmma implicit-GEMM convolutions, fused GroupNorm + SiLU, tensor-core attention GEMMs).  ``decode_to_uint8`` also
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
DECODER_PREFIXES = ("decoder.", "post_quant_conv.")
ENCODER_PREFIXES = ("encoder.", "quant_conv.")


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


def _mid_block(c):
    """UNetMidBlock2D of the decoder and the encoder: resnets.0, attentions.0 (one head of c channels), resnets.1."""
    mid = _Holder()
    att = _Holder()
    att.group_norm = nn.GroupNorm(32, c, eps=1e-6)
    att.to_q = nn.Linear(c, c)
    att.to_k = nn.Linear(c, c)
    att.to_v = nn.Linear(c, c)
    att.to_out = _List([nn.Linear(c, c)])
    mid.attentions = _List([att])
    mid.resnets = _List([_resnet(c, c), _resnet(c, c)])
    return mid


def _encoder(in_channels, boc, layers_per_block, latent_channels):
    """diffusers ``Encoder`` (double_z): conv_in, down blocks of ResnetBlock2D + Downsample2D(padding=0), the mid block,
    GroupNorm + SiLU + conv_out to 2 x latent_channels."""
    enc = _Holder()
    enc.conv_in = nn.Conv2d(in_channels, boc[0], 3, padding=1)
    downs, ch = [], boc[0]
    for i, out in enumerate(boc):
        blk = _Holder()
        res = []
        for _ in range(layers_per_block):
            res.append(_resnet(ch, out))
            ch = out
        blk.resnets = _List(res)
        if i != len(boc) - 1:
            down = _Holder()
            down.conv = nn.Conv2d(ch, ch, 3, stride=2, padding=0)
            blk.downsamplers = _List([down])
        downs.append(blk)
    enc.down_blocks = _List(downs)
    enc.mid_block = _mid_block(ch)
    enc.conv_norm_out = nn.GroupNorm(32, ch, eps=1e-6)
    enc.conv_out = nn.Conv2d(ch, 2 * latent_channels, 3, padding=1)
    return enc


class DiagonalGaussianDistribution:
    """diffusers ``DiagonalGaussianDistribution`` built from the moments the native encoder returns (logvar already clamped
    to [-30, 20]): ``std = exp(0.5 logvar)``, ``var = exp(logvar)``, ``sample(generator) = mean + std * eps``, ``mode() = mean``."""

    def __init__(self, mean, logvar):
        self.mean, self.logvar = mean, logvar
        self.std = torch.exp(0.5 * logvar)
        self.var = torch.exp(logvar)

    def sample(self, generator=None):
        """eps is drawn as diffusers' ``randn_tensor`` draws it: on the generator's device (the mean's when no generator is
        given), then moved to the mean's device.  On a CUDA generator the CUDA RNG stream advances exactly as under diffusers."""
        gen_dev = generator.device if generator is not None else self.mean.device
        eps = torch.randn(self.mean.shape, generator=generator, device=gen_dev, dtype=self.mean.dtype).to(self.mean.device)
        return self.mean + self.std * eps

    def mode(self):
        return self.mean


class _EncoderNative(_NativeNet):
    """The encoder's native context (lfm_create_vae_encoder): holds the AutoencoderKL's ``encoder`` and ``quant_conv``
    modules (shared, not copied), so its upload walks exactly their 108 keys.  Not a registered child of the AutoencoderKL."""

    def __init__(self, vae):
        super().__init__()
        self.encoder = vae.encoder
        self.quant_conv = vae.quant_conv
        self.block_out_channels, self.layers_per_block = vae.block_out_channels, vae.layers_per_block
        self.latent_channels, self.in_channels, self.norm_num_groups = vae.latent_channels, vae.in_channels, vae.norm_num_groups
        self.chunk_rule = vae.decode_chunk
        self._init_native()
        self._image_side = None

    def invalidate(self):
        """The AutoencoderKL's parameters may have changed or moved: redo the version walk on the next call."""
        self._dirty = True
        object.__setattr__(self, "_probe_cache", None)

    def latent_side(self):
        return self._image_side // 2 ** (len(self.block_out_channels) - 1)

    def _version(self):
        return (self._image_side,) + super()._version()

    def _create_ctx(self, lib, dev_index):
        boc = self.block_out_channels
        d = _lib.VaeDesc(self.latent_side(), self.latent_channels, self.in_channels, len(boc), (C.c_int32 * 8)(*boc),
                         self.layers_per_block, self.norm_num_groups)
        ctx = C.c_void_p()
        _lib.check(lib.lfm_create_vae_encoder(C.byref(d), dev_index, C.byref(ctx)))
        return ctx

    def _finalize_rows(self, rows):
        return max(rows, self.chunk_rule(self.latent_side()))


class AutoencoderKL(_NativeNet):
    """Mirror of ``diffusers.AutoencoderKL`` (defaults = the stabilityai/sd-vae-ft-mse config): the decoder, and with
    ``with_encoder=True`` the encoder as well (248 state-dict keys instead of 140)."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, norm_num_groups=32, scaling_factor=0.18215, max_batch=16, with_encoder=False, **unused):
        super().__init__()
        self.block_out_channels = tuple(int(c) for c in block_out_channels)
        self.layers_per_block, self.latent_channels, self.out_channels = int(layers_per_block), int(latent_channels), int(out_channels)
        self.in_channels = int(in_channels)
        self.norm_num_groups = int(norm_num_groups)
        self.with_encoder = bool(with_encoder)
        self.config = types.SimpleNamespace(scaling_factor=scaling_factor, block_out_channels=self.block_out_channels,
                                            layers_per_block=self.layers_per_block, latent_channels=self.latent_channels)
        self.max_batch_hint = max_batch
        if self.with_encoder:       # diffusers' registration order: encoder, decoder, quant_conv, post_quant_conv
            self.encoder = _encoder(self.in_channels, self.block_out_channels, self.layers_per_block, self.latent_channels)
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
        dec.mid_block = _mid_block(rev[0])
        dec.conv_norm_out = nn.GroupNorm(32, ch, eps=1e-6)
        dec.conv_out = nn.Conv2d(ch, out_channels, 3, padding=1)
        self.decoder = dec
        if self.with_encoder:
            self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.requires_grad_(False)
        self._init_native()
        self._latent_size = None
        # the encoder's own native context, not a registered child: the AutoencoderKL's state_dict is not doubled
        object.__setattr__(self, "_enc_native", _EncoderNative(self) if self.with_encoder else None)

    # -- loading ------------------------------------------------------------------------------------------------------
    @staticmethod
    def decoder_state_dict(sd):
        """The decoder entries of a (possibly full, possibly legacy-named) AutoencoderKL checkpoint."""
        return AutoencoderKL._select(sd, DECODER_PREFIXES)

    @staticmethod
    def _select(sd, prefixes):
        """The entries of `sd` under `prefixes`, legacy attention names renamed as diffusers does."""
        out = {}
        for k, v in sd.items():
            if not k.startswith(prefixes):
                continue
            parts = k.split(".")
            if "attentions" in parts and len(parts) >= 2 and parts[-2] in LEGACY_ATTN:
                parts[-2] = LEGACY_ATTN[parts[-2]]
                if v.dim() == 4:          # very old checkpoints store the projections as 1x1 convolutions
                    v = v[:, :, 0, 0]
            out[".".join(parts)] = v
        return out

    def load_state_dict(self, state_dict, strict=True, **kw):
        prefixes = DECODER_PREFIXES + (ENCODER_PREFIXES if self.with_encoder else ())
        r = super().load_state_dict(self._select(state_dict, prefixes), strict=strict, **kw)
        self._invalidate_encoder()
        return r

    def _invalidate_encoder(self):
        if getattr(self, "_enc_native", None) is not None:
            self._enc_native.invalidate()

    def mark_dirty(self):
        super().mark_dirty()
        self._invalidate_encoder()

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._invalidate_encoder()
        return r

    def _native_state_dict(self):
        return self.decoder_state_dict(self.state_dict())

    @classmethod
    def from_pretrained(cls, path, subfolder=None, with_encoder=False, **kwargs):
        """``AutoencoderKL.from_pretrained`` for a LOCAL diffusers directory (no hub access in this environment).
        ``with_encoder=True`` also loads the encoder (strictly: every ``encoder.*`` / ``quant_conv.*`` key must be there)."""
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
        vae = cls(**{k: cfg[k] for k in keep if k in cfg}, with_encoder=with_encoder, **kwargs)
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
        chunk = self.decode_chunk(h)
        ctx = self.native(min(B, chunk), z.device)
        lib = _lib.load()
        for i in range(0, B, chunk):
            n = min(chunk, B - i)
            _lib.check(lib.lfm_decode(ctx, z[i:i + n].data_ptr(), n, out[i:i + n].data_ptr() if want_f32 else None,
                                      u8[i:i + n].data_ptr() if want_u8 else None, self._stream(z.device)), ctx)
        return out, u8

    def decode_chunk(self, latent_side: int) -> int:
        """Images per native decode call, and the batch the native workspace is sized for: ``max_batch`` (default 16) for
        latents up to 32 x 32.  A 512 x 512 image (64 x 64 latents) needs four times the workspace of a 256 x 256 one, about
        1.2 GB per image, so there the chunk is ``max_batch // 4``: the same bytes as the 256-pixel decode at the same hint."""
        hint = max(1, int(self.max_batch_hint or 16))
        return max(1, hint // 4) if latent_side >= 64 else hint

    def _finalize_rows(self, rows):
        return max(rows, self.decode_chunk(self._latent_size))

    # -- first_stage_model.decode(z).sample  (test_flow_latent.py:193) --------------------------------------------------
    def decode(self, z, return_dict=True, **kwargs):
        sample, _ = self._decode_native(z, True, False)
        return types.SimpleNamespace(sample=sample) if return_dict else (sample,)

    def decode_to_uint8(self, z):
        """decode + ``(clamp((x + 1) / 2, 0, 1) * 255).permute(0, 2, 3, 1).to(uint8)`` (test_flow_latent_ddp.py:131-135)
        in one pass: [B, 4, s, s] latents -> [B, 8s, 8s, 3] uint8 on the device."""
        return self._decode_native(z, False, True)[1]

    # -- first_stage_model.encode(x).latent_dist  (downstream_tasks/test_flow_latent_inpainting.py:147) ----------------------
    def encode(self, x, return_dict=True):
        """x fp32 [B, 3, S, S] on a CUDA device (S = 128, 256 or 512) -> ``.latent_dist``, a DiagonalGaussianDistribution over
        [B, 4, S / 8, S / 8] latents (``(latent_dist,)`` with ``return_dict=False``).  Runs in chunks of ``decode_chunk``
        images, the decoder's rule at the same latent side."""
        if not self.with_encoder:
            raise RuntimeError("this AutoencoderKL holds the decoder only: build it with with_encoder=True "
                               "(AutoencoderKL(..., with_encoder=True) / from_pretrained(path, with_encoder=True))")
        if not x.is_cuda:
            raise RuntimeError("lfm_b200: x must be a CUDA tensor (no CPU path)")
        x = x.to(torch.float32).contiguous()
        B, Cc, h, w = x.shape
        down = 2 ** (len(self.block_out_channels) - 1)
        if Cc != self.in_channels or h != w or h % down != 0:
            raise ValueError(f"expected square images [B, {self.in_channels}, S, S] with S a multiple of {down}, got {tuple(x.shape)}")
        enc = self._enc_native
        if enc._image_side != h:
            enc._image_side = h
            enc.invalidate()                  # another image size = another native context
        s = h // down
        mean = torch.empty(B, self.latent_channels, s, s, device=x.device)
        logvar = torch.empty_like(mean)
        chunk = self.decode_chunk(s)
        ctx = enc.native(min(B, chunk), x.device)
        lib = _lib.load()
        for i in range(0, B, chunk):
            n = min(chunk, B - i)
            _lib.check(lib.lfm_encode(ctx, x[i:i + n].data_ptr(), n, mean[i:i + n].data_ptr(), logvar[i:i + n].data_ptr(),
                                      self._stream(x.device)), ctx)
        dist = DiagonalGaussianDistribution(mean, logvar)
        return types.SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    def forward(self, *a, **k):
        raise NotImplementedError("the native AutoencoderKL has no forward: use .decode(z) (and .encode(x) with with_encoder=True)")

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

    def encode_flops_per_image(self, image_side: int = 256) -> float:
        """Algorithmic FLOPs (2 x MAC) of one encode: the convolutions, quant_conv, the four attention projections and the
        two attention GEMMs."""
        boc, L2 = self.block_out_channels, 2 * self.latent_channels
        side, ch = image_side, boc[0]
        fl = 2.0 * side * side * 9 * self.in_channels * ch
        for i, out in enumerate(boc):
            px = side * side
            for _ in range(self.layers_per_block):
                fl += 2.0 * px * 9 * (ch * out + out * out) + (2.0 * px * ch * out if ch != out else 0.0)
                ch = out
            if i != len(boc) - 1:
                side //= 2
                fl += 2.0 * side * side * 9 * ch * ch
        px = side * side
        fl += 2 * (2.0 * px * 9 * 2 * ch * ch) + 2.0 * px * 4 * ch * ch + 4.0 * px * px * ch        # mid block
        return fl + 2.0 * px * (9 * ch * L2 + L2 * L2)


def synthetic_vae_state_dict(vae: AutoencoderKL, seed: int = 1):
    """Seeded non-degenerate weights for every key of `vae` (the decoder's, and the encoder's with with_encoder=True) (the real sd-vae-ft-mse file is a network download): conv / linear
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
