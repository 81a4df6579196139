"""Inpainting scores: FID, P-IDS and U-IDS between generated and ground-truth images, as the downstream readme computes them
with ``pytorch_fid/cal_inpainting.py <gen> <gt>`` (its ``calculate_metrics``).

    python -m lfm_b200.inpaint_metrics inpainting_generated_samples/celeba_256 gt_celeb --detector inception-2015-12-05.pt

The steps are the reference's:

1. Pairs: the ``*.png`` and ``*.jpg`` files of each directory, sorted by path; the ground truth is cut to its first 2950 files,
   and both lists must then be equally long.
2. Images: PNG decoded by pyspng when it imports, otherwise by PIL; JPEG by PIL without a mode conversion.  A one-channel
   image is repeated to three; the result is a uint8 ``[3, H, W]`` array, and the two images of a pair must share H and W.
3. Features: StyleGAN2-ADA's TorchScript Inception (``inception-2015-12-05.pt``, not the ``pt_inception-*.pth`` weights of
   ``lfm_b200.fid``), called as ``detector(img, return_features=True)``: 2048 fp32 features per image.  Every row is kept.
4. FID: fp64 sums of the features on the device (:class:`lfm_b200.fid.FIDStatistics`), the mean and the biased covariance
   ``sum(x x^T) / n - mu mu^T`` (the reference's ``FeatureStats``, not the n - 1 of ``fid_score.py``), and
   :func:`lfm_b200.fid.frechet_distance`.
5. P-IDS / U-IDS: ``sklearn.svm.LinearSVC(dual=False)`` fitted on the real rows (target 1) followed by the generated rows
   (target 0); U-IDS is its training error, P-IDS the fraction of pairs whose generated image gets the larger decision value.
6. ``fid: %.4f, pids: %.4f, uids: %.4f`` is printed and written to ``--out`` (default ``fid_pids_uids.txt``).

Two quirks of the reference are kept because they decide its numbers:
  * the 2950 cut: the CelebA-HQ evaluation set has 2993 ground-truth images, so the generated directory must hold exactly 2950
    (generate with ``--num_images 2950``);
  * the pairing is lexicographic, not numeric: the generator's ``0.jpg, 1.jpg, 10.jpg, 100.jpg, ...`` pair with
    ``000000.jpg, 000001.jpg, 000002.jpg, 000003.jpg, ...``.  P-IDS compares the SVM outputs of these pairs, so a generated
    image is mostly compared with the ground truth of another image.  FID and U-IDS do not depend on the pairing.

Differences, all deliberate:
  * the detector runs on batches of ``--batch-size`` images of one size (the reference calls it once per image), with TF32
    off so that the batch size cannot change the rounding of a convolution;
  * the paths, the output file and the detector file are arguments (the reference hard-codes them, ignores its command line
    and downloads the detector; there is no download here);
  * a ``ValueError`` is raised before the detector runs for unequal counts, a pair whose sizes differ, and an image that is
    not 1- or 3-channel (RGBA, LA, palette, CMYK), which the reference would pass on to the detector.
"""
from __future__ import annotations

import argparse
import glob
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import fid

GT_LIMIT = 2950
RESULT_FORMAT = "fid: %.4f, pids: %.4f, uids: %.4f"


def _linear_svc():
    try:
        from sklearn.svm import LinearSVC
    except ImportError as e:
        raise ImportError("the P-IDS / U-IDS step needs scikit-learn (sklearn.svm.LinearSVC, the reference's classifier); "
                          "install scikit-learn") from e
    return LinearSVC


def _device(device) -> torch.device:
    return torch.device(device if device else ("cuda" if torch.cuda.is_available() else "cpu"))


def _images_of(folder: str) -> List[str]:
    if not os.path.isdir(folder):
        raise FileNotFoundError(f"image directory not found: {folder}")
    return sorted(glob.glob(os.path.join(glob.escape(folder), "*.png")) + glob.glob(os.path.join(glob.escape(folder), "*.jpg")))


def _image_size(path: str) -> Tuple[int, int]:
    """(H, W) from the file's header; refuses what the reference's reader would not turn into three channels."""
    from PIL import Image
    with Image.open(path) as im:
        mode, (w, h), bands = im.mode, im.size, len(im.getbands())
    if mode in ("P", "PA") or bands not in (1, 3):
        raise ValueError(f"{path}: a {mode} image ({bands} channels); only 1- and 3-channel images are scored, "
                         "convert it to RGB first")
    return h, w


def image_pairs(gen_dir: str, gt_dir: str) -> Tuple[List[str], List[str], List[Tuple[int, int]]]:
    """Step 1 and the checks of step 2: the generated and ground-truth files in the reference's pairing, and the (H, W) of
    each pair.  Reads file headers only."""
    gen = _images_of(gen_dir)
    gt = _images_of(gt_dir)[:GT_LIMIT]
    if len(gen) != len(gt):
        raise ValueError(f"{gen_dir} holds {len(gen)} images and {gt_dir} {len(gt)} (the ground truth is cut to its first "
                         f"{GT_LIMIT}): the counts must be equal; generate with --num_images {GT_LIMIT}")
    if not gen:
        raise ValueError(f"no .png / .jpg images in {gen_dir} and {gt_dir}")
    sizes = []
    for a, b in zip(gen, gt):
        sa, sb = _image_size(a), _image_size(b)
        if sa != sb:
            raise ValueError(f"{a} is {sa[1]}x{sa[0]} but the ground truth it is paired with, {b}, is {sb[1]}x{sb[0]}")
        sizes.append(sa)
    return gen, gt, sizes


def _decode(path: str) -> np.ndarray:
    if path.endswith(".png"):
        try:
            import pyspng
        except ImportError:
            pyspng = None
        if pyspng is not None:
            with open(path, "rb") as f:
                return pyspng.load(f.read())
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im)


def read_image(path: str) -> np.ndarray:
    """Step 2: uint8 ``[3, H, W]``."""
    image = _decode(path)
    if image.ndim == 2:
        image = image[:, :, None]
    if image.shape[2] == 1:
        image = np.repeat(image, 3, axis=2)
    if image.shape[2] != 3:
        raise ValueError(f"{path}: decoded to {image.shape[2]} channels; only 1- and 3-channel images are scored")
    return image.transpose(2, 0, 1).astype(np.uint8)


def load_detector(path: str, device=None) -> torch.jit.ScriptModule:
    """``path``: a local copy of StyleGAN2-ADA's ``inception-2015-12-05.pt`` (there is no download)."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f"detector file not found: {path} (there is no network access; pass a local copy of "
                                "inception-2015-12-05.pt)")
    return torch.jit.load(path, map_location=device).eval()


@torch.no_grad()
def detector_features(detector, files: Sequence[str], sizes: Sequence[Tuple[int, int]], batch_size: int,
                      device) -> Tuple[torch.Tensor, fid.FIDStatistics]:
    """Step 3 and the sums of step 4: every feature row (``[n, D]`` fp32 on ``device``, in the order of ``files``) and their
    fp64 statistics.  Consecutive images of one size share a detector call, at most ``batch_size`` of them; TF32 is off
    during the calls, so that the batch size does not decide whether a convolution rounds its operands to TF32."""
    rows, stats = [], None
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        i = 0
        while i < len(files):
            j = i + 1
            while j < len(files) and j - i < batch_size and sizes[j] == sizes[i]:
                j += 1
            x = torch.from_numpy(np.stack([read_image(f) for f in files[i:j]])).to(device)
            f = detector(x, return_features=True).to(torch.float32)
            if f.dim() != 2 or f.shape[0] != j - i:
                raise ValueError(f"the detector returned {tuple(f.shape)} features for {j - i} images; expected [{j - i}, D]")
            if stats is None:
                stats = fid.FIDStatistics(f.shape[1], device)
            stats.update(f)
            rows.append(f)
            i = j
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    return torch.cat(rows), stats


def mean_cov(stats: fid.FIDStatistics) -> Tuple[torch.Tensor, torch.Tensor]:
    """The reference's ``FeatureStats.get_mean_cov``: the mean and the biased (/n) covariance."""
    mu = stats.s1 / stats.n
    return mu, stats.s2 / stats.n - torch.outer(mu, mu)


def pids_uids(real: np.ndarray, fake: np.ndarray) -> Tuple[float, float]:
    """Step 5 on the fp32 feature rows of the ground truth and of the generated images, paired row for row."""
    svm = _linear_svc()(dual=False)
    inputs = np.concatenate([real, fake])
    targets = np.array([1] * real.shape[0] + [0] * fake.shape[0])
    svm.fit(inputs, targets)
    uids = 1 - svm.score(inputs, targets)
    pids = np.mean(svm.decision_function(fake) > svm.decision_function(real))
    return float(pids), float(uids)


def inpainting_metrics(gen_dir: str, gt_dir: str, detector, batch_size: int = 50, device=None) -> Tuple[float, float, float]:
    """(fid, pids, uids) of the generated images in ``gen_dir`` against the ground truth in ``gt_dir``.  ``detector`` is the
    loaded TorchScript Inception (:func:`load_detector`), or any callable with its signature, on ``device``."""
    if batch_size < 1:
        raise ValueError(f"batch size must be >= 1, got {batch_size}")
    device = _device(device)
    _linear_svc()         # fail before the feature pass, not after it
    gen, gt, sizes = image_pairs(gen_dir, gt_dir)
    fake, fake_stats = detector_features(detector, gen, sizes, batch_size, device)
    real, real_stats = detector_features(detector, gt, sizes, batch_size, device)
    mu1, sigma1 = mean_cov(fake_stats)
    mu2, sigma2 = mean_cov(real_stats)
    fid_value = fid.frechet_distance(mu1, sigma1, mu2, sigma2, device=device)
    pids, uids = pids_uids(real.cpu().numpy(), fake.cpu().numpy())
    return fid_value, pids, uids


def build_parser():
    p = argparse.ArgumentParser("python -m lfm_b200.inpaint_metrics",
                                description="FID, P-IDS and U-IDS between generated inpainting results and the ground truth")
    p.add_argument("gen", nargs="?", default="./inpainting_generated_samples/celeba_256/", help="generated images")
    p.add_argument("gt", nargs="?", default="./gt_celeb/", help=f"ground-truth images (the first {GT_LIMIT} are used)")
    p.add_argument("--detector", type=str, required=True,
                   help="local copy of StyleGAN2-ADA's inception-2015-12-05.pt (there is no download)")
    p.add_argument("--out", type=str, default="fid_pids_uids.txt", help="file the result line is written to")
    p.add_argument("--batch-size", type=int, default=50, help="images per detector call")
    p.add_argument("--device", type=str, default=None, help="cuda, cuda:N or cpu (default: cuda when available)")
    return p


def main(argv: Optional[Sequence[str]] = None) -> Tuple[float, float, float]:
    args = build_parser().parse_args(argv)
    device = _device(args.device)
    detector = load_detector(args.detector, device)
    fid_value, pids, uids = inpainting_metrics(args.gen, args.gt, detector, args.batch_size, device)
    line = RESULT_FORMAT % (fid_value, pids, uids)
    print(line)
    with open(args.out, "w") as f:
        f.write(line)
    return fid_value, pids, uids


if __name__ == "__main__":
    main()
