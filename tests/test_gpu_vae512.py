"""The 512 x 512 VAE decode (64 x 64 latents, the celeb512 preset) on the H100 (`-m gpu`): its kernels at the new sizes, the whole
decode against the oracle, the command line at --image_size 512, and the 128 / 256 pixel decodes left bit-identical.

Kernel bounds are those of tests/test_gpu_kernels.py (see its header), which also supplies the GroupNorm and batched-GEMM checks:
  * 3x3 convolution, fp32 out: |y - ref| <= (K + 16) 2^-23 (|A| * |W| + |bias| + |out_0|) elementwise and rel-L2 <= 1e-5 (K <= 2304
    here); bf16 out: one bf16 ulp more.  The 512-pixel rows run on four 128-pixel segments, so the columns on both sides of the three
    inner seams (127 / 128, 255 / 256, 383 / 384) read their left / right neighbours from the next segment's box, and the first and
    last row and column read the TMA's zero fill: those columns and rows are also checked on their own, where a seam read as padding
    (an error of ~sqrt(3 Cin) |a| |w|, hundreds of times the bound) cannot be diluted by the rest of the image.
  * GroupNorm statistics of the conv epilogue at 2^20 values per (image, group): half a fixed-point unit per add plus the conv's
    own bound carried into the sums; at rms 1000 the sum of squares (1.0e12 per group) is 1/8 of the 2^43 the bins hold.

End-to-end decode against oracle/vae.py run on the GPU in fp32 with TF32 off (and with its bf16 operand emulation).  Measured on an
H100 80GB HBM3 (latent 64, B = 3, synthetic weights seed 1): native vs fp32 oracle rel-L2 1.70e-2, the bf16-emulating oracle 1.51e-2
(the 256-pixel decode: about 1.5e-2 both), so the bounds of test_vae_decode_vs_oracle carry over: 3e-2 absolute, 1.25 x the noise floor
+ 1e-3 relative.  uint8 images at most 8 grey levels from the oracle's, as far as the emulation's; 4.9 % of the pixels off by more than one
level, 0.72 % by more than two.
"""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lfm_b200
from lfm_b200 import _lib
from tests import test_gpu_kernels as tk

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEAM_COLS = [0, 1, 127, 128, 255, 256, 383, 384, 510, 511]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------ convolution at side 512


def conv_ref_rows(x, w, bias, rows=64):
    """fp64 conv2d (pad 1, stride 1) of NHWC bf16 operands as an im2col matmul in slabs of `rows` output rows: the value and the
    conv of the absolute values."""
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    xp = F.pad(x.double(), (0, 0, 1, 1, 1, 1))
    wd = w.double().t()                                            # [9 Cin, Cout], K index (r * 3 + s) * Cin + c
    wa = wd.abs()
    y = torch.empty(B, H, W, Cout, dtype=torch.float64, device=x.device)
    ya = torch.empty_like(y)
    for b in range(B):
        for h0 in range(0, H, rows):
            cols = torch.cat([xp[b, h0 + r:h0 + r + rows, s:s + W] for r in range(3) for s in range(3)], -1).reshape(-1, 9 * Cin)
            y[b, h0:h0 + rows] = (cols @ wd).reshape(rows, W, Cout)
            ya[b, h0:h0 + rows] = (cols.abs() @ wa).reshape(rows, W, Cout)
    return y + bias.double(), ya + bias.double().abs()


def run_conv_wide(x, w, bias, out, block_n, epi, bins=None):
    B, side, _, Cin = x.shape
    rc = _lib.load().lfm_dbg_conv_wide(tk.P(x), tk.P(w), tk.P(bias), tk.P(out), tk.P(bins), B, side, Cin, w.shape[0], 1, block_n, epi,
                                       1, None)
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()


def check_wide(out, ref, absref, K, what, out0=None):
    """tk.check_conv on the whole output, then on the seam columns and the edge rows alone."""
    tk.check_conv(out, ref, absref, K, what, out0)
    side = out.shape[1]
    cols = [c for c in SEAM_COLS if c < side] if side == 512 else [0, 1, 127, 128, side - 2, side - 1]
    o0c = out0[:, :, cols] if out0 is not None else None
    tk.check_conv(out[:, :, cols], ref[:, :, cols], absref[:, :, cols], K, what + " seam / edge columns", o0c)
    o0r = out0[:, [0, side - 1]] if out0 is not None else None
    tk.check_conv(out[:, [0, side - 1]], ref[:, [0, side - 1]], absref[:, [0, side - 1]], K, what + " first / last row", o0r)


# (side, Cin, Cout, B): the decoder's 512-pixel stage pairs them as up_blocks.2 conv2 / upsampler (256 -> 256), up_blocks.3
# resnets.0 conv1 (256 -> 128), the rest of up_blocks.3 (128 -> 128); one 256-pixel case (two segments per row)
WIDE = [(512, 256, 256, 1), (512, 256, 256, 3), (512, 256, 128, 1), (512, 256, 128, 3), (512, 128, 128, 1), (512, 128, 128, 3),
        (256, 128, 128, 3)]


@pytest.mark.parametrize("side,Cin,Cout,B", WIDE)
def test_conv3x3_wide_rows(dev, side, Cin, Cout, B):
    x, w, bias = tk.conv_operands(B, side, Cin, Cout, side + 7 * Cin + Cout + B)
    ref, absref = conv_ref_rows(x, w, bias)
    K = 9 * Cin
    out0 = torch.randn(B, side, side, Cout, generator=torch.Generator().manual_seed(B + Cout)).cuda()
    for block_n in (128, 256):
        out = torch.full((B, side, side, Cout), float("nan"), device=dev)
        run_conv_wide(x, w, bias, out, block_n, 3)
        check_wide(out, ref, absref, K, f"conv {side} {Cin}->{Cout} B{B} bn{block_n}")
        outb = torch.full((B, side, side, Cout), float("nan"), device=dev).bfloat16()
        run_conv_wide(x, w, bias, outb, block_n, 0)
        check_wide(outb, ref, absref, K, f"bf16 conv {side} {Cin}->{Cout} B{B} bn{block_n}")
        acc = out0.clone()
        run_conv_wide(x, w, bias, acc, block_n, 2)
        check_wide(acc, out0.double() + ref, absref, K, f"residual conv {side} {Cin}->{Cout} B{B} bn{block_n}", out0=out0)
        del out, outb, acc


@pytest.mark.parametrize("block_n", [128, 256])
@pytest.mark.parametrize("Cin,Cout,B,rms,epi", [
    (256, 128, 2, 1.0, 3),      # cpg 4, 2^20 values per group
    (128, 128, 1, 1000.0, 0),   # sum of squares ~1e12 per group, bf16 store
    (256, 256, 1, 1.0, 0),      # cpg 8
    (256, 256, 1, 1000.0, 3),
])
def test_conv_wide_groupnorm_statistics(dev, Cin, Cout, B, rms, epi, block_n):
    side = 512
    x, w, bias = tk.conv_operands(B, side, Cin, Cout, Cin + Cout + B, w_std=rms * (9 * Cin) ** -0.5)
    bias = bias * rms
    ref, absref = conv_ref_rows(x, w, bias)
    bins = [torch.zeros(B * tk.REPLICAS * 64, dtype=torch.int64, device=dev) for _ in range(2)]
    out = torch.full((B, side, side, Cout), float("nan"), device=dev)
    if epi == 0:
        out = out.bfloat16()
    for bb in bins:
        run_conv_wide(x, w, bias, out, block_n, epi, bb)
    assert torch.equal(bins[0], bins[1]), "statistics bins differ between two identical calls"
    check_wide(out, ref, absref, 9 * Cin, "conv with statistics")
    S, Q = tk.bins_to_stats(bins[0], B)
    cpg, HW = Cout // 32, side * side
    rg = ref.reshape(B, HW, 32, cpg)
    S_ref, Q_ref = rg.sum((1, 3)), (rg * rg).sum((1, 3))
    adds = HW // 16
    err_y = (tk.dot_c(9 * Cin) * absref).reshape(B, HW, 32, cpg)
    S_bound = adds * 0.5 / tk.GN_SCALE + err_y.sum((1, 3)) + 16 * cpg * 2.0 ** -24 * rg.abs().sum((1, 3))
    Q_bound = adds * 0.5 / tk.GN_SCALE_SQ + (2 * rg.abs() * err_y + err_y ** 2).sum((1, 3)) + 16 * cpg * 2.0 ** -24 * Q_ref
    tk.assert_within(S, S_ref, S_bound, "group sum")
    tk.assert_within(Q, Q_ref, Q_bound, "group sum of squares")
    assert float(Q_ref.max()) < 2.0 ** 43       # inside the fixed-point range (rms < 2896 at 2^20 values per group)


# ------------------------------------------------------------------------------------------------ GroupNorm at 512 x 512

# (Ca, Cb, HW, B, eps, film, act, source, max_chunks, copy_out, raw_out, mean / std) as tk.GN_CASES: the decoder's 512-pixel stage
GN512 = [
    (128, 0, 262144, 1, 1e-6, None, 1, "f32", 256, True, True, 0),    # 256-chunk fp64 statistics pass, SiLU, both side outputs
    (256, 0, 262144, 2, 1e-6, None, 1, "f32", 256, False, True, 0),   # the upsampler output feeding up_blocks.3, + raw_out
    (256, 0, 262144, 1, 1e-6, None, 0, "f32", 256, True, False, 0),   # no SiLU, copy_out
    (128, 0, 262144, 2, 1e-6, None, 1, "bins", 32, True, False, 0),   # statistics from bins, fp32 source, copy_out
    (128, 0, 262144, 1, 1e-6, None, 1, "bf16", 32, False, False, 0),  # conv1 output as bf16 with bins: the fast path, J = 1
    (256, 0, 262144, 1, 1e-6, None, 1, "bf16", 32, False, True, 0),   # bf16 source with raw_out: the generic pass, J = 2
]


@pytest.mark.parametrize("Ca,Cb,HW,B,eps,film,act,source,max_chunks,copy,raw,mean", GN512)
def test_groupnorm_512(dev, Ca, Cb, HW, B, eps, film, act, source, max_chunks, copy, raw, mean):
    tk.test_groupnorm(dev, Ca, Cb, HW, B, eps, film, act, source, max_chunks, copy, raw, mean)


# ------------------------------------------------------------------------------------------------ mid-block attention at 4096 tokens


@pytest.mark.parametrize("B", [1, 2])
def test_vae_attention_batched_gemms_4096(dev, B):
    """V^T, S = Q K^T (fp32, 4096 x 4096 per image) and O = P V + b at 64 x 64 latents, C = 512."""
    tk.test_vae_attention_batched_gemms(dev, 4096, B)


# ------------------------------------------------------------------------------------------------ end-to-end decode


def oracle_on_gpu(sd, z, dev, emulate_bf16=False):
    from oracle import vae as ovae
    tf = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        out = ovae.vae_decode({k: v.to(dev) for k, v in sd.items()}, z.to(dev), emulate_bf16=emulate_bf16)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf
    return out.cpu()


def test_vae_decode_512_vs_oracle(dev):
    """AutoencoderKL.decode at 64 x 64 latents (512 x 512 images), 3 images with max_batch 8: decode chunks of two images (the
    workspace of a 512-pixel image is four times that of a 256-pixel one, so the chunk is max_batch // 4), the last chunk odd."""
    from oracle import vae as ovae
    vae = lfm_b200.AutoencoderKL(max_batch=8)
    sd = ovae.synthetic_state_dict(ovae.VAEConfig(), 1)
    vae.load_state_dict(sd, strict=True)
    vae = vae.to(dev).eval()
    assert vae.decode_chunk(64) == 2
    B, side = 3, 64
    z = torch.randn(B, 4, side, side, generator=torch.Generator().manual_seed(164)) / 0.18215 * 0.2
    out = vae.decode(z.to(dev)).sample
    assert out.shape == (B, 3, 512, 512) and torch.isfinite(out).all()
    ref = oracle_on_gpu(sd, z, dev)
    emu = oracle_on_gpu(sd, z, dev, emulate_bf16=True)
    err, noise_floor = tk.rel_l2(out.cpu(), ref), tk.rel_l2(emu, ref)
    print(f"\n512 decode: native vs fp32 oracle rel-L2 {err:.4g}, bf16-emulating oracle {noise_floor:.4g}")
    assert err < 3e-2
    assert err < 1.25 * noise_floor + 1e-3, (err, noise_floor)
    assert torch.equal(out, vae.decode(z.to(dev)).sample)                          # deterministic
    assert tk.rel_l2(vae.decode(z[2:].to(dev)).sample.cpu(), out[2:].cpu()) < 1e-5    # samples are independent
    u8 = vae.decode_to_uint8(z.to(dev))
    assert u8.dtype == torch.uint8 and u8.shape == (B, 512, 512, 3)
    assert torch.equal(u8.cpu(), ovae.to_uint8_nhwc(out.cpu()))
    d = (u8.cpu().int() - ovae.to_uint8_nhwc(ref).int()).abs()
    d_emu = int((ovae.to_uint8_nhwc(emu).int() - ovae.to_uint8_nhwc(ref).int()).abs().max())
    print(f"grey levels: max {int(d.max())} (emulation {d_emu}), >1: {float((d > 1).float().mean()):.4f}, "
          f">2: {float((d > 2).float().mean()):.4f}")
    assert int(d.max()) <= max(8, d_emu + 1) and float((d > 1).float().mean()) < 0.08 and float((d > 2).float().mean()) < 0.01


def test_vae_512_max_batch_beyond_the_upsampler_grid_is_refused(dev):
    """max_batch 1024 at 64 x 64 latents sizes the context for 256 images; the last upsampler would need 256 x 256 = 65536 grid
    rows, one more than a launch allows: lfm_finalize refuses it, saying why, before it allocates anything."""
    vae = lfm_b200.AutoencoderKL(max_batch=1024)
    vae.load_state_dict(lfm_b200.synthetic_vae_state_dict(vae, 1), strict=True)
    vae = vae.to(dev).eval()
    with pytest.raises(RuntimeError, match=r"max_batch 256 is too large.*max_batch <= 255"):
        vae.decode(torch.zeros(1, 4, 64, 64, device=dev))


# ------------------------------------------------------------------------------------------------ command line at 512


def test_cli_decodes_512_images(dev, tmp_path):
    """test_flow_latent.py at --image_size 512 (64 x 64 latents) with the native decoder: the generation loop writes 512 x 512
    JPEGs under the reference's file indices, the default mode writes the image grid, and the device FID runs on them."""
    from PIL import Image
    from lfm_b200 import cli
    out = str(tmp_path)
    common = ["--model_type", "DiT-B/2", "--image_size", "512", "--num_in_channels", "4", "--num_classes", "1", "--label_dropout", "0.",
              "--method", "euler", "--step_size", "0.5", "--synthetic_init", "3", "--synthetic_vae", "2", "--out_dir", out,
              "--device", "cuda:0", "--dataset", "celeba_256", "--exp", "t"]
    assert cli.main(common + ["--batch_size", "1", "--n_sample", "2", "--compute_fid"]) == 0
    d = os.path.join(out, "generated_samples", "celeba_256", "expt_ep1000_meuler_s40")
    files = sorted(os.listdir(d), key=lambda f: int(f.split(".")[0]))
    assert files == ["0.jpg", "1.jpg"]
    imgs = [np.asarray(Image.open(os.path.join(d, f))) for f in files]
    assert all(im.shape == (512, 512, 3) and im.std() > 1.0 for im in imgs)
    assert cli.main(common + ["--batch_size", "2"]) == 0
    assert Image.open(os.path.join(out, "samples_celeba_256_euler_1e-05_1e-05.jpg")).size == (1024, 512)
    stat, log = os.path.join(out, "stat.npy"), os.path.join(out, "fid.log")
    feats = np.random.RandomState(0).rand(64, 2048)
    np.save(stat, {"mu": feats.mean(0), "sigma": np.cov(feats, rowvar=False)}, allow_pickle=True)
    assert cli.main(common + ["--batch_size", "2", "--n_sample", "2", "--compute_fid", "--synthetic_inception", "1", "--no_save",
                              "--real_img_dir", stat, "--output_log", log, "--dataset", "custom"]) == 0
    value = float(open(log).read().strip().split("FID = ")[1])
    assert np.isfinite(value) and value > 0


# ------------------------------------------------------------------------------------------------ smaller decodes unchanged


def load_recipe():
    spec = importlib.util.spec_from_file_location("make_vae_golden", os.path.join(ROOT, "scripts", "make_vae_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_decode_16_and_32_bit_identical_to_the_recorded_fingerprint(dev):
    """The decodes at latent 16 and 32 (128 / 256 pixel images) give the very bytes recorded from the build before the 512-pixel
    decode existed (tests/golden/vae_decode_fingerprint.npz, scripts/make_vae_golden.py)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "vae_decode_fingerprint.npz"))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if sms != int(g["num_sms"]):
        pytest.skip(f"fingerprint recorded with {int(g['num_sms'])} SMs ({g['device']}); the split-K plan differs on {sms}")
    recipe = load_recipe()
    for side, B, mb in recipe.CASES:
        got = recipe.fingerprint(side, B, mb, dev)
        sub, want = got[f"s{side}_f32_sub"], g[f"s{side}_f32_sub"]
        assert got[f"s{side}_f32_sha256"] == str(g[f"s{side}_f32_sha256"]), \
            f"latent {side}: fp32 sample differs, max |diff| in the subsample {float(np.abs(sub - want).max()):.3g}"
        assert got[f"s{side}_u8_sha256"] == str(g[f"s{side}_u8_sha256"]), f"latent {side}: uint8 image differs"
