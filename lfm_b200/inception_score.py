"""Inception Score on the device: ``pytorch_fid/inception_score.py`` without TensorFlow (SURVEY.md 8(f)-4).

``python -m lfm_b200.inception_score --sample_dir samples.npy --inception_weights pt_inception-2015-12-05-6726825d.pth``
prints the reference's three lines (``Calculating Inception Score with N images in S splits``, ``mean: ``, ``std: ``);
``--compute_fid --compute_is`` on the sampling command line (lfm_b200/cli.py) scores the generated images in the loop.

What the reference computes, and this module too:

1. ``x / 255 * 2 - 1`` on ``[N, 3, H, W]`` values in 0..255, then TF1's legacy ``resize_bilinear`` to 299 x 299
   (:func:`prepare_tf1`: no corner alignment, no half-pixel centres, source coordinate ``dst * (in / out)`` in fp32,
   neighbours ``floor`` and ``min(floor + 1, in - 1)``).  It is not the half-pixel resize of ``FIDInception.prepare``.
2. The class logits of the 2015-12-05 Inception graph, ``[:, :1000]``, and their softmax in fp32.  TF-GAN's
   ``inception/1`` TF-Hub module is that frozen graph and its ``logits`` output is ``softmax/logits``, the layer the
   published ``pt_inception-2015-12-05-6726825d.pth`` carries as ``fc.weight`` / ``fc.bias``; so the network here is
   :class:`~lfm_b200.fid.FIDInception` (the FID trunk) built ``with_logits``.  That equivalence is not verified: this
   project does not use TensorFlow and no test compares the two.
3. Per split ``s`` of ``n_s`` images, ``IS_s = exp(mean_i KL(p_i || mean_i p_i))``; ``mean`` and population ``std`` over
   the splits.  :class:`ISStatistics` keeps, per split and in fp64 on the device, ``n_s``, ``P_s = sum_i p_i`` and
   ``H_s = sum_i sum_c p_ic log p_ic``, so ``IS_s = exp((H_s - sum_c P_sc log(P_sc / n_s)) / n_s)``: the same sum
   regrouped so that batches stream in any order and ranks combine with ONE all-reduce of an ``[S, 1002]`` buffer.
   The reference's split ``i`` is the rows ``i * N // S .. (i + 1) * N // S - 1``, so image ``k`` belongs to split
   ``((k + 1) * S - 1) // N`` (the largest ``i`` with ``i * N // S <= k``; ``k * S // N`` differs when ``S`` does
   not divide ``N``, e.g. ``k = 9`` for ``N = 37, S = 4``).

Deviations, both deliberate:

* The softmax subtracts the row maximum.  The reference's ``exp(l) / sum(exp(l))`` gives the same numbers except
  where its ``exp`` overflows (a logit above ~88 in fp32) and it returns ``inf`` / ``nan``.  ``0 log 0`` counts as 0;
  the reference's ``p * log(p)`` is ``nan`` for a probability that underflowed to zero.
* In the generation loop the score comes from the decoder's uint8 images; the reference scores an ``.npy`` built from
  the JPEG files, so its number includes the JPEG compression (as for FID, lfm_b200/fid.py).
"""
from __future__ import annotations

import argparse
import os
import pathlib
from typing import List, Tuple

import numpy as np
import torch

from . import fid as lfid

NUM_CLASSES = 1000     # logits[:, :1000] (inception_score.py:77): the graph's 1008 outputs include 8 unused classes


def _tf1_axis(n_in: int, n_out: int, device):
    """TF1 legacy bilinear weights along one axis: source ``dst * (in / out)`` in fp32, lower / upper neighbour, lerp."""
    scale = torch.tensor(float(n_in), dtype=torch.float32) / n_out
    src = torch.arange(n_out, dtype=torch.float32) * scale
    lo = src.floor()
    i0 = lo.long()
    i1 = (i0 + 1).clamp_max(n_in - 1)
    return i0.to(device), i1.to(device), (src - lo).to(device)


def prepare_tf1(images: torch.Tensor) -> torch.Tensor:
    """uint8 ``[B, H, W, 3]`` (the decoder's output) or float ``[B, 3, H, W]`` in 0..255 -> ``[B, 3, 299, 299]`` fp32
    in [-1, 1]: ``x / 255 * 2 - 1`` then ``tf.compat.v1.image.resize_bilinear`` (inception_score.py:52, 74), on the
    tensor's device.  Rows and columns are interpolated as TF's kernel does: across first, then down."""
    if images.dtype == torch.uint8:
        if images.dim() != 4 or images.shape[-1] != 3:
            raise ValueError(f"uint8 images must be [B, H, W, 3], got {tuple(images.shape)}")
        x = images.permute(0, 3, 1, 2).float()
    else:
        if images.dim() != 4 or images.shape[1] != 3:
            raise ValueError(f"float images must be [B, 3, H, W], got {tuple(images.shape)}")
        x = images.float()
    x = x / 255.0 * 2 - 1
    y0, y1, ly = _tf1_axis(x.shape[2], 299, x.device)
    x0, x1, lx = _tf1_axis(x.shape[3], 299, x.device)

    def across(rows):
        left, right = rows.index_select(3, x0), rows.index_select(3, x1)
        return left + (right - left) * lx
    top, bottom = across(x.index_select(2, y0)), across(x.index_select(2, y1))
    return top + (bottom - top) * ly[:, None]


def inception_probs(net: lfid.FIDInception, images: torch.Tensor, batch: int = 64) -> torch.Tensor:
    """``[B, 1000]`` fp32 class probabilities of a batch (uint8 NHWC or float NCHW in 0..255, see :func:`prepare_tf1`):
    the legacy resize, the FID trunk and ``fc`` on ``images``' device, in chunks of ``batch`` images
    (inception_score.py:69-79; the softmax subtracts the row maximum, see the module docstring)."""
    out = [torch.softmax(net.logits(prepare_tf1(images[i:i + batch]))[:, :NUM_CLASSES], dim=1)
           for i in range(0, images.shape[0], batch)]
    return torch.cat(out, 0)


class ISStatistics:
    """Per-split sums of the Inception Score over ``n`` images in ``splits`` splits, fp64 on ``device``: one row per split
    of ``[n_s, P_s (1000), H_s]``.  ``update(probs, first_index, stride)`` takes the probabilities of images
    ``first_index + j * stride``; ``all_reduce`` sums the ranks; ``scores`` / ``finalize`` give the per-split scores and
    ``(mean, std)``."""

    def __init__(self, splits: int, n: int, device=None):
        if splits < 1:
            raise ValueError(f"splits must be >= 1, got {splits}")
        if splits > n:
            raise ValueError(f"{splits} splits of {n} images: every split needs at least one image")
        self.splits, self.n = int(splits), int(n)
        self.buf = torch.zeros(self.splits, NUM_CLASSES + 2, dtype=torch.float64, device=device)

    def split_of(self, index: torch.Tensor) -> torch.Tensor:
        """The split of image ``index``: the one whose rows ``i * n // S .. (i + 1) * n // S - 1`` hold it
        (inception_score.py:85)."""
        return ((index + 1) * self.splits - 1) // self.n

    def update(self, probs: torch.Tensor, first_index: int, stride: int = 1) -> None:
        if probs.dim() != 2 or probs.shape[1] != NUM_CLASSES:
            raise ValueError(f"probabilities must be [B, {NUM_CLASSES}], got {tuple(probs.shape)}")
        if self.buf.device != probs.device:
            self.buf = self.buf.to(probs.device)
        last = first_index + stride * (probs.shape[0] - 1)
        if first_index < 0 or last >= self.n:
            raise ValueError(f"image indices {first_index} .. {last} are outside 0 .. {self.n - 1}")
        index = first_index + stride * torch.arange(probs.shape[0], device=probs.device)
        p = probs.double()
        rows = torch.cat([torch.ones_like(p[:, :1]), p, torch.xlogy(p, p).sum(1, keepdim=True)], 1)
        self.buf.index_add_(0, self.split_of(index), rows)

    def all_reduce(self) -> None:
        """Sum over the ranks of the default process group: one collective on the ``[S, 1002]`` buffer."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.buf)

    def scores(self) -> torch.Tensor:
        """``[S]`` fp64: ``exp((H_s - sum_c P_sc log(P_sc / n_s)) / n_s)``."""
        n, p, h = self.buf[:, 0], self.buf[:, 1:-1], self.buf[:, -1]
        if bool((n < 1).any()):
            raise ValueError(f"split image counts {n.tolist()}: every split needs at least one image")
        return torch.exp((h - torch.xlogy(p, p / n[:, None]).sum(1)) / n)

    def finalize(self) -> Tuple[float, float]:
        """``(np.mean, np.std)`` of the per-split scores (inception_score.py:89; population std)."""
        s = self.scores()
        return float(s.mean()), float(s.std(correction=0))


# ---------------------------------------------------------------------------------------------------------------------
# the reference's script (inception_score.py:108-118), on an .npy array or an image directory
# ---------------------------------------------------------------------------------------------------------------------
def list_images_in_order(path: str) -> List[pathlib.Path]:
    """The images of a directory (``fid.list_images``), by integer stem when every stem is an integer (the sampling
    command lines write ``{index}.jpg``) and by name otherwise."""
    files = lfid.list_images(path)
    if files and all(f.stem.isdigit() for f in files):
        files = sorted(files, key=lambda f: int(f.stem))
    return files


def check_array(data: np.ndarray) -> None:
    """get_inception_score's checks (inception_score.py:94-96) as ValueError: ``[N, 3, H, W]`` with values in 0..255,
    which the first image's maximum above 10 is taken to show (arrays scaled to [0, 1] are refused)."""
    if data.ndim != 4 or data.shape[1] != 3:
        raise ValueError(f"images must be an [N, 3, H, W] array, got shape {data.shape}")
    if data.shape[0] == 0:
        raise ValueError("the array holds no images")
    if not (np.min(data[0]) >= 0 and np.max(data[0]) > 10):
        raise ValueError("Image values should be in the range [0, 255]")


def _directory_batches(files, batch_size, device):
    from PIL import Image
    for i in range(0, len(files), batch_size):
        batch = [np.asarray(Image.open(f).convert("RGB")) for f in files[i:i + batch_size]]
        sizes = sorted({b.shape for b in batch})
        if len(sizes) > 1:
            raise ValueError(f"images of one batch differ in size ({', '.join(f'{h}x{w}' for h, w, _ in sizes)}), "
                             f"from {files[i].name}")
        yield i, torch.from_numpy(np.stack(batch)).to(device)


def build_parser():
    p = argparse.ArgumentParser("python -m lfm_b200.inception_score", description="Inception Score of generated images")
    p.add_argument("--sample_dir", type=str, default="./saved_samples/",
                   help="an .npy of [N, 3, H, W] values in 0..255, or a directory of images")
    p.add_argument("--inception_weights", type=str, required=True,
                   help="local copy of pt_inception-2015-12-05-6726825d.pth, fc layer included (there is no download)")
    p.add_argument("--splits", type=int, default=1, help="number of splits (the reference's script uses 1)")
    p.add_argument("--batch-size", type=int, default=64, help="images per network call")
    p.add_argument("--device", type=str, default=None, help="cuda, cuda:N or cpu (default: cuda when available)")
    return p


def main(argv=None) -> Tuple[float, float]:
    args = build_parser().parse_args(argv)
    if args.splits < 1:
        raise ValueError(f"--splits must be >= 1, got {args.splits}")
    if args.batch_size < 1:
        raise ValueError(f"--batch-size must be >= 1, got {args.batch_size}")
    device = torch.device(args.device if args.device else ("cuda" if torch.cuda.is_available() else "cpu"))
    if os.path.isdir(args.sample_dir):
        files = list_images_in_order(args.sample_dir)
        n = len(files)
        batches = _directory_batches(files, args.batch_size, device)
    elif os.path.isfile(args.sample_dir):
        data = np.clip(np.load(args.sample_dir), 0, 255)          # inception_score.py:113-114
        check_array(data)
        n = data.shape[0]
        batches = ((i, torch.from_numpy(np.asarray(data[i:i + args.batch_size], dtype=np.float32)).to(device))
                   for i in range(0, n, args.batch_size))
    else:
        raise RuntimeError("Invalid path: %s" % args.sample_dir)
    stats = ISStatistics(args.splits, n, device)                   # refuses splits > n before the network runs
    net =lfid.FIDInception.from_file(args.inception_weights, with_logits=True).to(device).eval()
    print("Calculating Inception Score with %i images in %i splits" % (n, args.splits))
    for first, images in batches:
        stats.update(inception_probs(net, images, args.batch_size), first)
    mean, std = stats.finalize()
    print("mean: ", mean)
    print("std: ", std)
    return mean, std


if __name__ == "__main__":
    main()
