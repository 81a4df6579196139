"""lfm_b200.inpaint_metrics on the CPU: FID, P-IDS and U-IDS between two image directories against the restated reference
(tests/tools/inpaint_metrics_oracle.py), its pairing, its 2950 cut, its refusals, batching and output.

The detector is a stand-in with the signature of StyleGAN2-ADA's TorchScript Inception: ``forward(img: uint8 [B, 3, H, W],
return_features=False, ...) -> [B, D]``, seeded convolutions after a float cast and a (x - 128) / 128 shift, saved with
``torch.jit.script`` and loaded from the file as the real one is.  By default it computes in fp64 and returns fp32, so that
its features do not depend on how many images share a call: the oracle's one-image calls and the module's batches then give
the same fp32 rows, and the metrics can be compared exactly.  ``dtype=torch.float32`` gives an fp32 detector like the real one.
"""
import os
import re
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from lfm_b200 import inpaint_metrics as im
from tests.tools import inpaint_metrics_oracle as oracle

pytestmark = pytest.mark.filterwarnings("ignore:`torch.jit:DeprecationWarning")


class StandInDetector(torch.nn.Module):
    def __init__(self, dims: int, seed: int, dtype: torch.dtype):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.w1 = torch.nn.Parameter((torch.randn(16, 3, 3, 3, generator=g) / 27 ** 0.5).to(dtype), requires_grad=False)
        self.b1 = torch.nn.Parameter((0.1 * torch.randn(16, generator=g)).to(dtype), requires_grad=False)
        self.w2 = torch.nn.Parameter((torch.randn(32, 16, 3, 3, generator=g) / 144 ** 0.5).to(dtype), requires_grad=False)
        # scaled so that FIDs of the test images are O(1), printed with a few significant digits
        self.w3 = torch.nn.Parameter((4 * torch.randn(dims, 32, 1, 1, generator=g)).to(dtype), requires_grad=False)

    def forward(self, img: torch.Tensor, return_features: bool = False, use_fp16: bool = False,
                no_output_bias: bool = False) -> torch.Tensor:
        x = img.to(self.w1.dtype)
        x = F.interpolate(x, size=(32, 32), mode="bilinear", align_corners=False)
        x = (x - 128) / 128
        x = F.relu(F.conv2d(x, self.w1, self.b1, stride=2))
        x = F.relu(F.conv2d(x, self.w2, stride=2))
        f = F.conv2d(x, self.w3).mean(dim=(2, 3)).to(torch.float32)
        return f if return_features else torch.softmax(f, 1)


def save_detector(path, dims=16, seed=3, dtype=torch.float64):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")              # torch.jit is deprecated on torch 2.11 but works
        torch.jit.script(StandInDetector(dims, seed, dtype)).save(str(path))
    return str(path)


def load_detector(path, device="cpu"):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return im.load_detector(str(path), torch.device(device))


@pytest.fixture
def detector_file(tmp_path):
    return save_detector(tmp_path / "det16.pt")


def raising_detector(*args, **kwargs):
    raise AssertionError("the detector must not be called")


def smooth_image(rng, h, w, gray=False):
    c = 1 if gray else 3
    low = torch.from_numpy(rng.uniform(0, 255, (1, c, max(2, h // 6), max(2, w // 6))))
    x = F.interpolate(low, size=(h, w), mode="bilinear", align_corners=False)[0].permute(1, 2, 0)
    a = x.round().clamp(0, 255).to(torch.uint8).numpy()
    return a[..., 0] if gray else a


def write_set(root, n=40, seed=0, size=(32, 32), gray_jpeg=(5,), gray_png=(12,)):
    """The inpainting command line's layout: ``gen/{i}.jpg`` and ground truth ``gt/{i:06d}.jpg``, generated image i being
    ground truth i with a rectangle repainted.  Generated images in ``gray_jpeg`` are grayscale JPEGs, ground-truth images in
    ``gray_png`` grayscale PNGs (and their generated counterparts grayscale too)."""
    rng = np.random.default_rng(seed)
    gen, gt = root / "gen", root / "gt"
    gen.mkdir(parents=True)
    gt.mkdir(parents=True)
    h, w = size
    for i in range(n):
        gray = i in gray_jpeg or i in gray_png
        real = smooth_image(rng, h, w, gray)
        fake = real.copy()
        y0, x0 = rng.integers(0, h // 2), rng.integers(0, w // 2)
        fake[y0:y0 + h // 2, x0:x0 + w // 2] = smooth_image(rng, h // 2, w // 2, gray)
        Image.fromarray(real).save(gt / (f"{i:06d}.png" if i in gray_png else f"{i:06d}.jpg"))
        Image.fromarray(fake).save(gen / f"{i}.jpg")
    return str(gen), str(gt)


def test_listing_pairs_lexicographically(tmp_path):
    gen, gt = write_set(tmp_path, n=13)
    g, t, sizes = im.image_pairs(gen, gt)
    assert [os.path.basename(p) for p in g] == ["0.jpg", "1.jpg", "10.jpg", "11.jpg", "12.jpg"] + [f"{i}.jpg" for i in range(2, 10)]
    assert [os.path.basename(p) for p in t] == [f"{i:06d}.jpg" for i in range(12)] + ["000012.png"]
    assert sizes == [(32, 32)] * 13
    for path in (os.path.join(gen, "5.jpg"), os.path.join(gt, "000012.png")):
        gray = im.read_image(path)
        assert gray.shape == (3, 32, 32) and gray.dtype == np.uint8
        assert np.array_equal(gray[0], np.array(Image.open(path))) and np.array_equal(gray[0], gray[2])


def test_metrics_match_oracle(tmp_path, detector_file):
    gen, gt = write_set(tmp_path)
    det = load_detector(detector_file)
    got = im.inpainting_metrics(gen, gt, det, batch_size=8, device="cpu")
    want = oracle.inpainting_metrics(gen, gt, det)
    assert got[0] > 0 and abs(got[0] - want[0]) <= 1e-9 * want[0]
    assert got[1:] == want[1:]
    assert 0 < got[2] < 0.5                          # 80 rows in 16 dimensions: not separable


def test_metrics_match_oracle_rank_deficient(tmp_path):
    """40 images, 64 features: both covariances are singular; scipy's sqrtm goes complex and the reference keeps its real
    part, the eigh route clamps the negative round-off eigenvalues (lfm_b200.fid.frechet_distance).  Each of the 24 null
    directions leaves a square root of fp64 noise, about 2^-26 lambda_max, in either route, so the agreement is bounded
    relative to lambda_max / FID, which is ~4 here: 9e-8 measured.  The bound is tests/test_fid.py's for its singular case."""
    gen, gt = write_set(tmp_path, seed=1)
    det = load_detector(save_detector(tmp_path / "det64.pt", dims=64, seed=4))
    got = im.inpainting_metrics(gen, gt, det, batch_size=16, device="cpu")
    want = oracle.inpainting_metrics(gen, gt, det)
    assert abs(got[0] - want[0]) <= 1e-6 * want[0]
    assert got[1:] == want[1:]


def test_pairing_is_lexicographic_not_numeric(tmp_path, detector_file):
    """P-IDS compares the SVM outputs of the pairs in sorted path order: generated 10.jpg against 000002.jpg, and so on."""
    gen, gt = write_set(tmp_path, seed=2)
    det = load_detector(detector_file)
    got = im.inpainting_metrics(gen, gt, det, batch_size=8, device="cpu")
    fake, real = oracle.features(gen, gt, det)
    want = oracle.scores(fake, real)
    assert abs(got[0] - want[0]) <= 1e-9 * want[0] and got[1:] == want[1:]
    numeric = np.argsort([int(os.path.basename(p)[:-4]) for p in oracle.listing(gen)])
    fid_n, pids_n, uids_n = oracle.scores(fake[numeric], real)
    assert pids_n != got[1]                          # the numeric pairing would print another P-IDS
    assert abs(fid_n - got[0]) <= 1e-9 * got[0] and uids_n == got[2]      # FID and U-IDS do not depend on it


def test_ground_truth_is_cut_to_2950(tmp_path, detector_file):
    rng = np.random.default_rng(5)
    gen, gt = tmp_path / "gen", tmp_path / "gt"
    gen.mkdir()
    gt.mkdir()
    for i in range(im.GT_LIMIT + 1):
        Image.fromarray(rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)).save(gt / f"{i:06d}.png")
    for i in range(im.GT_LIMIT):
        Image.fromarray(rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)).save(gen / f"{i}.png")
    g, t, _ = im.image_pairs(str(gen), str(gt))
    assert len(g) == len(t) == 2950 and os.path.basename(t[-1]) == "002949.png"
    det = load_detector(detector_file)
    fid_value, pids, uids = im.inpainting_metrics(str(gen), str(gt), det, batch_size=500, device="cpu")
    assert fid_value > 0 and 0 <= pids <= 1 and 0 < uids < 1

    Image.fromarray(rng.integers(0, 256, (8, 8, 3), dtype=np.uint8)).save(gen / f"{im.GT_LIMIT}.png")
    with pytest.raises(ValueError, match=r"2951 images .* 2950 .*--num_images 2950"):
        im.inpainting_metrics(str(gen), str(gt), raising_detector, device="cpu")


def test_refusals_come_before_the_detector(tmp_path, detector_file):
    gen, gt = write_set(tmp_path, n=6)

    def refused(exc, match):
        with pytest.raises(exc, match=match):
            im.inpainting_metrics(gen, gt, raising_detector, device="cpu")

    Image.fromarray(smooth_image(np.random.default_rng(0), 32, 40)).save(os.path.join(gen, "3.jpg"))
    refused(ValueError, r"3\.jpg is 40x32 but .*000003\.jpg, is 32x32")
    Image.fromarray(smooth_image(np.random.default_rng(0), 32, 32)).save(os.path.join(gen, "3.jpg"))

    rgba = np.concatenate([smooth_image(np.random.default_rng(1), 32, 32), np.full((32, 32, 1), 255, np.uint8)], 2)
    os.remove(os.path.join(gt, "000004.jpg"))
    Image.fromarray(rgba).save(os.path.join(gt, "000004.png"))
    refused(ValueError, r"000004\.png: a RGBA image \(4 channels\)")
    Image.fromarray(smooth_image(np.random.default_rng(1), 32, 32)).convert("P").save(os.path.join(gt, "000004.png"))
    refused(ValueError, r"000004\.png: a P image")
    Image.fromarray(smooth_image(np.random.default_rng(1), 32, 32)).convert("CMYK").save(os.path.join(gen, "4.jpg"))
    refused(ValueError, r"4\.jpg: a CMYK image \(4 channels\)")
    Image.fromarray(smooth_image(np.random.default_rng(1), 32, 32)).save(os.path.join(gen, "4.jpg"))
    Image.fromarray(smooth_image(np.random.default_rng(1), 32, 32)).save(os.path.join(gt, "000004.png"))
    assert len(im.image_pairs(gen, gt)[0]) == 6

    with pytest.raises(FileNotFoundError, match="missing"):
        im.inpainting_metrics(gen, str(tmp_path / "missing"), raising_detector, device="cpu")
    with pytest.raises(FileNotFoundError, match=r"nope\.pt"):
        im.main([gen, gt, "--detector", str(tmp_path / "nope.pt"), "--out", str(tmp_path / "out.txt"), "--device", "cpu"])
    empty_a, empty_b = tmp_path / "ea", tmp_path / "eb"
    empty_a.mkdir()
    empty_b.mkdir()
    with pytest.raises(ValueError, match="no .png / .jpg images"):
        im.inpainting_metrics(str(empty_a), str(empty_b), raising_detector, device="cpu")
    with pytest.raises(ValueError, match="batch size"):
        im.inpainting_metrics(gen, gt, raising_detector, batch_size=0, device="cpu")
    assert not (tmp_path / "out.txt").exists()


def test_batch_size_changes_no_result(tmp_path):
    """An fp32 detector, as the real one, and pairs of three sizes so that the batches break at the size changes."""
    rng = np.random.default_rng(7)
    gen, gt = tmp_path / "gen", tmp_path / "gt"
    gen.mkdir()
    gt.mkdir()
    sizes = [(32, 32)] * 9 + [(24, 40)] * 4 + [(32, 32)] * 11 + [(48, 48)] * 6
    names = sorted(f"{i}.jpg" for i in range(len(sizes)))
    for r, (h, w) in enumerate(sizes):
        Image.fromarray(smooth_image(rng, h, w, gray=r == 3)).save(gen / names[r])
        Image.fromarray(smooth_image(rng, h, w)).save(gt / f"{r:06d}.jpg")
    det = load_detector(save_detector(tmp_path / "det32.pt", dtype=torch.float32))
    g, _, s = im.image_pairs(str(gen), str(gt))
    assert s == sizes
    f1, _ = im.detector_features(det, g, s, 1, "cpu")
    f7, st7 = im.detector_features(det, g, s, 7, "cpu")
    with torch.no_grad():
        per_image = torch.cat([det(torch.from_numpy(im.read_image(p))[None], return_features=True) for p in g])
    assert float((f1 - per_image).norm() / per_image.norm()) <= 1e-6
    assert float((f7 - per_image).norm() / per_image.norm()) <= 1e-6
    assert st7.n == len(sizes) and torch.allclose(st7.s1, f7.double().sum(0), rtol=1e-12, atol=0)

    out = str(tmp_path / "out.txt")
    common = [str(gen), str(gt), "--detector", str(tmp_path / "det32.pt"), "--out", out, "--device", "cpu"]
    m1 = im.main(common + ["--batch-size", "1"])
    m7 = im.main(common + ["--batch-size", "7"])
    assert m1[1:] == m7[1:] and abs(m1[0] - m7[0]) <= 1e-5 * m1[0]
    assert im.RESULT_FORMAT % m1 == im.RESULT_FORMAT % m7


def test_output_line(tmp_path, detector_file, capsys):
    gen, gt = write_set(tmp_path, n=20, seed=3)
    out = tmp_path / "scores" / "fid_pids_uids.txt"
    out.parent.mkdir()
    got = im.main([gen, gt, "--detector", detector_file, "--out", str(out), "--batch-size", "6", "--device", "cpu"])
    printed = capsys.readouterr().out
    line = out.read_text()
    assert printed == line + "\n"
    assert re.fullmatch(r"fid: \d+\.\d{4}, pids: \d\.\d{4}, uids: \d\.\d{4}", line)
    assert line == "fid: %.4f, pids: %.4f, uids: %.4f" % got
    assert isinstance(got, tuple) and all(isinstance(v, float) for v in got)


def test_command_line_without_a_detector(tmp_path, capsys):
    with pytest.raises(SystemExit) as e:
        im.main(["--help"])
    assert e.value.code == 0
    help_text = capsys.readouterr().out
    assert "--detector" in help_text and "--batch-size" in help_text and "--out" in help_text
    with pytest.raises(SystemExit) as e:
        im.main([str(tmp_path), str(tmp_path)])
    assert e.value.code == 2 and "--detector" in capsys.readouterr().err
    args = im.build_parser().parse_args(["--detector", "d.pt"])
    assert (args.gen, args.gt, args.out, args.batch_size) == ("./inpainting_generated_samples/celeba_256/", "./gt_celeb/",
                                                              "fid_pids_uids.txt", 50)


def test_missing_sklearn_is_an_error(tmp_path, monkeypatch):
    gen, gt = write_set(tmp_path, n=4)
    monkeypatch.setitem(__import__("sys").modules, "sklearn.svm", None)
    with pytest.raises(ImportError, match="P-IDS / U-IDS step needs scikit-learn"):
        im.inpainting_metrics(gen, gt, raising_detector, device="cpu")
    with pytest.raises(ImportError, match="P-IDS / U-IDS"):
        im.pids_uids(np.zeros((4, 3), np.float32), np.ones((4, 3), np.float32))
