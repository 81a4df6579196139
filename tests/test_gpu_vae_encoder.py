"""The native VAE encoder (AutoencoderKL.encode, the inpainting loop's first step) on the H100 (`-m gpu`): its new kernels against
fp64, the whole encode against the oracle (tests/tools/vae_encoder_oracle.py), the distribution's sample, and the inpainting
command line end to end.

Kernel bounds are those of tests/test_gpu_kernels.py (see its header):
  * Downsample2D(padding=0), the stride-2 convolution with tap origin 0: fp32 out within (K + 16) 2^-23 (|A| * |W| + |bias|)
    elementwise, K = 9 Cin, and rel-L2 <= 1e-5; bf16 out one bf16 ulp more.  The bottom row and the right column read the
    tensor map's zero fill in place of F.pad's extra line, and at 512 -> 256 the 256-column box of a row segment ends past the
    image and the columns 127 / 128 meet at the seam: those lines are also checked on their own, where a tap read one pixel
    off (an error of ~sqrt(3 Cin) |a| |w|) cannot be diluted by the rest of the image.
  * conv_in at 3 channels (fp32 operands): (K + 16) 2^-23 (|x| * |w| + |bias|), K = 27.
  * vae_quant_kernel: 16 2^-24 (sum |w| |x| + |b|) for mean and logvar, the clamp at both bounds exact.

End to end against the oracle run on the GPU in fp32 with TF32 off, and with its bf16 operand emulation: the encoder amplifies the
operand rounding as the decoder does, so the bounds are the decoder's, rel-L2 < 3e-2 and <= 1.25 x (emulated vs fp32 oracle)
+ 1e-3, for mean and logvar.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lfm_b200
from lfm_b200 import _lib
from tests import test_gpu_kernels as tk
from tests.tools import vae_encoder_oracle as oenc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------ Downsample2D(padding=0)


def conv_down_ref(x, w, bias):
    """fp64 conv2d(F.pad(x, (0, 1, 0, 1)), stride=2) on the bf16 operands, NHWC: the value and the conv of the absolute values."""
    Cout, Cin = w.shape[0], x.shape[-1]
    xd = F.pad(x.double().permute(0, 3, 1, 2), (0, 1, 0, 1))
    wd = w.double().reshape(Cout, 3, 3, Cin).permute(0, 3, 1, 2)     # K index (r * 3 + s) * Cin + c
    y = F.conv2d(xd, wd, stride=2).permute(0, 2, 3, 1) + bias.double()
    ya = F.conv2d(xd.abs(), wd.abs(), stride=2).permute(0, 2, 3, 1) + bias.double().abs()
    return y, ya


# (input side, Cin, B): the encoder's three downsamplers at 256 pixels, and the first one at 512 pixels (row segments)
DOWN = [(256, 128, 2), (128, 256, 2), (64, 512, 3), (512, 128, 1)]


@pytest.mark.parametrize("epi", [3, 0])   # fp32 out (the network's), bf16 out
@pytest.mark.parametrize("side,Cin,B", DOWN)
def test_conv_down_vs_fp64(dev, side, Cin, B, epi):
    x, w, bias = tk.conv_operands(B, side, Cin, Cin, seed=side + Cin + epi)
    o = side // 2
    out = torch.empty(B, o, o, Cin, device=dev, dtype=torch.float32 if epi == 3 else torch.bfloat16)
    rc = _lib.load().lfm_dbg_conv_down(tk.P(x), tk.P(w), tk.P(bias), tk.P(out), None, B, side, Cin, Cin, 2, 0, epi, -1 if epi == 3 else 1,
                                       None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    ref, absref = conv_down_ref(x, w, bias)
    K = 9 * Cin
    tk.check_conv(out, ref, absref, K, f"down {side} -> {o}, Cin {Cin}")
    lines = {"bottom row": (slice(None), o - 1), "right column": (slice(None), slice(None), o - 1)}
    if o > 128:
        lines.update({"seam column 127": (slice(None), slice(None), 127), "seam column 128": (slice(None), slice(None), 128)})
    for what, idx in lines.items():
        tk.check_conv(out[idx], ref[idx], absref[idx], K, f"down {side}: {what}")
    # a pad-1 convolution of the same operands differs: the tap origin is really 0
    assert tk.rel_l2(out, tk.conv_ref(x, w, bias, 2)[0]) > 0.1


# ------------------------------------------------------------------------------------------------ conv_in at 3 channels


@pytest.mark.parametrize("side", [256, 512])
def test_conv_in_3_channels(dev, side):
    g = torch.Generator().manual_seed(side)
    B, Cout = 2, 128
    x = (torch.rand(B, 3, side, side, generator=g) * 2 - 1).to(dev)
    w = (torch.randn(Cout, 3, 3, 3, generator=g) / 5).to(dev)
    bias = torch.randn(Cout, generator=g).to(dev)
    out = torch.empty(B, side, side, Cout, device=dev)
    _lib.check(_lib.load().lfm_dbg_conv_in(tk.P(x), 3, 3 * side * side, None, 0, 0, tk.P(w), tk.P(bias), tk.P(out), B, side, Cout, None))
    torch.cuda.synchronize()
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(x.double().abs(), w.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    tk.assert_within(out, ref, (27 + 16) * 2.0 ** -23 * mag, f"conv_in 3 -> {Cout} at {side}")


# ------------------------------------------------------------------------------------------------ quant_conv + moments


def test_vae_quant_kernel(dev):
    g = torch.Generator().manual_seed(9)
    B, HW = 3, 32 * 32
    x = torch.randn(B * HW, 8, generator=g) * 4
    w = torch.randn(8, 8, generator=g)
    b = torch.randn(8, generator=g)
    x[:50, 4:] = 40.0          # logvar far above 20 on some pixels, far below -30 on others
    x[50:100, 4:] = -40.0
    w[4:, 4:] = torch.eye(4) * 2
    x, w, b = x.to(dev), w.to(dev), b.to(dev)
    mean = torch.empty(B, 4, HW, device=dev)
    logvar = torch.empty_like(mean)
    _lib.check(_lib.load().lfm_dbg_vae_quant(tk.P(x), tk.P(w), tk.P(b), tk.P(mean), tk.P(logvar), B, HW, None))
    torch.cuda.synchronize()
    y = (x.double() @ w.double().t() + b.double()).reshape(B, HW, 8).permute(0, 2, 1)
    mag = (x.double().abs() @ w.double().abs().t() + b.double().abs()).reshape(B, HW, 8).permute(0, 2, 1)
    bound = 16 * 2.0 ** -24 * mag
    tk.assert_within(mean, y[:, :4], bound[:, :4], "mean")
    ref_lv = y[:, 4:].clamp(-30, 20)
    tk.assert_within(logvar, ref_lv, bound[:, 4:], "logvar")
    assert (logvar == 20.0).sum() > 0 and (logvar == -30.0).sum() > 0
    assert torch.equal(logvar[y[:, 4:] > 21], torch.full_like(logvar[y[:, 4:] > 21], 20.0))
    assert torch.equal(logvar[y[:, 4:] < -31], torch.full_like(logvar[y[:, 4:] < -31], -30.0))


# ------------------------------------------------------------------------------------------------ end-to-end encode


def oracle_on_gpu(sd, x, dev, emulate_bf16=False):
    tf = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        m, lv = oenc.vae_encode({k: v.to(dev) for k, v in sd.items()}, x.to(dev), emulate_bf16=emulate_bf16)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf
    return m.cpu(), lv.cpu()


def images(B, side, seed):
    """Smooth images in [-1, 1] with some texture: bilinear upsampling of a coarse random field plus noise."""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand(B, 3, side // 16, side // 16, generator=g) * 2 - 1
    x = F.interpolate(coarse, size=(side, side), mode="bilinear", align_corners=False)
    return (x + 0.1 * torch.randn(B, 3, side, side, generator=g)).clamp(-1, 1)


@pytest.fixture(scope="module")
def weights():
    return oenc.synthetic_state_dict(seed=1)


@pytest.mark.parametrize("side,B,max_batch", [(128, 3, 16), (256, 2, 1), (512, 1, 4)])
def test_encode_vs_oracle(dev, weights, side, B, max_batch):
    vae = lfm_b200.AutoencoderKL(with_encoder=True, max_batch=max_batch)
    vae.load_state_dict(weights, strict=True)
    vae = vae.to(dev).eval()
    x = images(B, side, side)
    dist = vae.encode(x.to(dev)).latent_dist
    s = side // 8
    assert dist.mean.shape == dist.logvar.shape == (B, 4, s, s)
    ref_m, ref_lv = oracle_on_gpu(weights, x, dev)
    emu_m, emu_lv = oracle_on_gpu(weights, x, dev, emulate_bf16=True)
    for name, got, ref, emu in (("mean", dist.mean, ref_m, emu_m), ("logvar", dist.logvar, ref_lv, emu_lv)):
        err, noise = tk.rel_l2(got.cpu(), ref), tk.rel_l2(emu, ref)
        print(f"\nencode {side} px, B {B}: {name} native vs fp32 oracle rel-L2 {err:.4g}, bf16-emulating oracle {noise:.4g}")
        assert err < 3e-2, (name, err)
        assert err < 1.25 * noise + 1e-3, (name, err, noise)
    again = vae.encode(x.to(dev)).latent_dist
    assert torch.equal(again.mean, dist.mean) and torch.equal(again.logvar, dist.logvar)            # deterministic
    one = vae.encode(x[B - 1:].to(dev)).latent_dist                                                  # images are independent
    assert tk.rel_l2(one.mean, dist.mean[B - 1:]) < 1e-5 and tk.rel_l2(one.logvar, dist.logvar[B - 1:]) < 1e-5
    (d2,) = vae.encode(x.to(dev), return_dict=False)
    assert torch.equal(d2.mean, dist.mean)


def test_sample_is_mean_plus_std_eps(dev, weights):
    vae = lfm_b200.AutoencoderKL(with_encoder=True, max_batch=2)
    vae.load_state_dict(weights, strict=True)
    vae = vae.to(dev).eval()
    dist = vae.encode(images(2, 128, 3).to(dev)).latent_dist
    assert torch.equal(dist.mode(), dist.mean)
    assert torch.equal(dist.std, torch.exp(0.5 * dist.logvar)) and torch.equal(dist.var, torch.exp(dist.logvar))
    state = torch.cuda.get_rng_state(dev)
    s = dist.sample()
    torch.cuda.set_rng_state(state, dev)
    eps = torch.randn(dist.mean.shape, device=dev, dtype=dist.mean.dtype)
    assert torch.equal(s, dist.mean + torch.exp(0.5 * dist.logvar) * eps)
    g = torch.Generator(device=dev).manual_seed(11)
    s = dist.sample(generator=g)
    eps = torch.randn(dist.mean.shape, generator=torch.Generator(device=dev).manual_seed(11), device=dev)
    assert torch.equal(s, dist.mean + dist.std * eps)


def test_mid_block_attention_is_live(dev, weights):
    """Zeroing the encoder's attention output projection changes the native mean as it changes the oracle's."""
    x = images(1, 128, 21)
    cut = dict(weights)
    cut["encoder.mid_block.attentions.0.to_out.0.weight"] = torch.zeros_like(weights["encoder.mid_block.attentions.0.to_out.0.weight"])
    cut["encoder.mid_block.attentions.0.to_out.0.bias"] = torch.zeros_like(weights["encoder.mid_block.attentions.0.to_out.0.bias"])
    vae = lfm_b200.AutoencoderKL(with_encoder=True, max_batch=1)
    vae.load_state_dict(weights, strict=True)
    vae = vae.to(dev).eval()
    full = vae.encode(x.to(dev)).latent_dist.mean.cpu()
    vae.load_state_dict(cut, strict=True)        # the encoder's context is re-uploaded
    zeroed = vae.encode(x.to(dev)).latent_dist.mean.cpu()
    d_native = full - zeroed
    d_oracle = oracle_on_gpu(weights, x, dev)[0] - oracle_on_gpu(cut, x, dev)[0]
    rel = tk.rel_l2(d_native, d_oracle)
    print(f"\nattention's share of the mean: {float(d_oracle.norm() / full.norm()):.3g}; native vs oracle change rel-L2 {rel:.3g}")
    assert float(d_native.norm()) > 0.5 * float(d_oracle.norm()) > 0
    assert rel < 0.3


def test_round_trip_256(dev, weights):
    vae = lfm_b200.AutoencoderKL(with_encoder=True, max_batch=2)
    vae.load_state_dict(weights, strict=True)
    vae = vae.to(dev).eval()
    z = vae.encode(images(2, 256, 5).to(dev)).latent_dist.mode()
    assert z.shape == (2, 4, 32, 32)
    img = vae.decode(z).sample
    assert img.shape == (2, 3, 256, 256) and torch.isfinite(img).all()
    with pytest.raises(RuntimeError, match="lfm_decode"):     # each context refuses the other's call
        _lib.check(_lib.load().lfm_decode(vae._enc_native._ctx, tk.P(z), 1, tk.P(img), None, None))
    with pytest.raises(RuntimeError, match="lfm_encode"):
        _lib.check(_lib.load().lfm_encode(vae._ctx, tk.P(img), 1, tk.P(z), tk.P(z), None))


def test_contexts_refuse_each_others_keys(dev):
    import ctypes as C
    lib = _lib.load()
    desc = _lib.VaeDesc(16, 4, 3, 4, (C.c_int32 * 8)(128, 256, 512, 512), 2, 32)
    w = torch.zeros(8, 8, 1, 1)
    shape = (C.c_int64 * 4)(8, 8, 1, 1)
    for create, key in ((lib.lfm_create_vae, b"quant_conv.weight"), (lib.lfm_create_vae_encoder, b"post_quant_conv.weight")):
        ctx = C.c_void_p()
        _lib.check(create(C.byref(desc), 0, C.byref(ctx)))
        try:
            assert lib.lfm_set_param(ctx, key, C.c_void_p(w.data_ptr()), 0, shape, 4) != 0
            assert "unexpected key" in _lib.last_error(ctx)
        finally:
            lib.lfm_destroy(ctx)


# ------------------------------------------------------------------------------------------------ inpainting command line


def write_dataset(root, n, side=256):
    from PIL import Image
    gt, masks = root / "gt", root / "masks"
    gt.mkdir()
    masks.mkdir()
    rng = np.random.default_rng(1)
    for i in range(n):
        img = (images(1, side, 40 + i)[0].permute(1, 2, 0).numpy() * 127.5 + 127.5).astype(np.uint8)
        Image.fromarray(img).save(gt / f"{i:06d}.jpg")
        m = np.full((side, side), 255, np.uint8)
        y0, x0 = rng.integers(32, 128, 2)
        m[y0:y0 + 96, x0:x0 + 80] = 0                      # the hole
        Image.fromarray(m).save(masks / f"{i:06d}.png")
    return str(gt), str(masks)


def test_inpainting_cli(dev, tmp_path):
    """test_flow_latent_inpainting.py with synthetic weights, the reference's inpainting UNet flags, batch 2, Euler at step 0.25
    on two images: the JPEGs under the reference's names, the batch equal to the same steps composed from the library calls,
    and the pixels outside the hole the input image's."""
    from lfm_b200 import cli_inpaint
    from lfm_b200.downstream import WrapperCondFlow, sample_from_model
    gt, masks = write_dataset(tmp_path, 2)
    argv = ["--batch_size", "2", "--method", "euler", "--step_size", "0.25", "--synthetic_init", "1", "--synthetic_vae", "2",
            "--gt_dir", gt, "--mask_dir", masks, "--num_images", "2", "--num_workers", "0", "--out_dir", str(tmp_path),
            "--device", "cuda:0", "--seed", "7"]
    assert cli_inpaint.main(argv) == 0
    d = tmp_path / "inpainting_generated_samples" / "celeba_256"
    assert sorted(os.listdir(d)) == ["0.jpg", "1.jpg"]
    from PIL import Image
    assert all(Image.open(d / f).size == (256, 256) for f in ("0.jpg", "1.jpg"))

    args = cli_inpaint.build_parser().parse_args(argv)
    model, vae = cli_inpaint.load(args, dev)
    ds = cli_inpaint.InpaintingEvalDataset(gt, masks, 2)
    image, mask, masked = (torch.stack(t).to(dev) for t in zip(ds[0], ds[1]))

    torch.manual_seed(7)
    torch.cuda.manual_seed_all(7)
    u8 = cli_inpaint.inpaint(args, model, vae, image, mask, masked)

    torch.manual_seed(7)
    torch.cuda.manual_seed_all(7)
    c = vae.encode(masked).latent_dist.sample() * args.scale_factor
    c = torch.cat((c, F.interpolate(mask, size=c.shape[-2:])), dim=1)
    z_0 = torch.randn(2, 4, 32, 32).to(dev)
    fake = sample_from_model(WrapperCondFlow(model, c), z_0, args)[-1]
    fake_image = (vae.decode(fake / args.scale_factor).sample + 1) / 2
    m = (mask + 1) / 2
    x = fake_image * m + (1 - m) * (image + 1) / 2
    hand = (x * 255 + 0.5).clamp(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert u8.shape == (2, 256, 256, 3)
    assert torch.equal(u8, hand)

    outside = (m[:, 0] == 0)
    want = torch.round((image + 1) / 2 * 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert int(outside.sum()) > 0 and int((~outside).sum()) > 0
    assert torch.equal(u8[outside], want[outside])
    assert float((u8[~outside].float() - want[~outside].float()).abs().mean()) > 1.0   # the hole is filled, not copied
