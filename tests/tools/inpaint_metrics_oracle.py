"""Test oracle for lfm_b200.inpaint_metrics: the downstream readme's inpainting score (FID, P-IDS, U-IDS between a generated and
a ground-truth directory) restated step for step in numpy / scipy / sklearn, one detector call per image in pair order.

``detector`` is any callable taking a uint8 ``[1, 3, H, W]`` tensor (and ``return_features=True``) and returning ``[1, D]``
features; ``device`` is where the images are sent before the call."""
import glob

import numpy as np
import scipy.linalg
import sklearn.svm
import torch
from PIL import Image


def listing(folder):
    return sorted(glob.glob(folder + "/*.png") + glob.glob(folder + "/*.jpg"))


def read(path):
    try:
        import pyspng
    except ImportError:
        pyspng = None
    if pyspng is not None and path.endswith(".png"):
        with open(path, "rb") as f:
            a = pyspng.load(f.read())
    else:
        a = np.array(Image.open(path))
    if a.ndim == 2:
        a = a[..., None]
    if a.shape[2] == 1:
        a = np.concatenate([a] * 3, axis=2)
    return torch.from_numpy(np.ascontiguousarray(a.transpose(2, 0, 1)))[None].to(torch.uint8)


def features(gen_dir, gt_dir, detector, device="cpu"):
    """(fake [n, D], real [n, D]) fp32 numpy rows in the reference's pairing."""
    gen, gt = listing(gen_dir), listing(gt_dir)[:2950]
    assert len(gen) == len(gt), (len(gen), len(gt))
    fake, real = [], []
    with torch.no_grad():
        for a, b in zip(gen, gt):
            x, y = read(a).to(device), read(b).to(device)
            assert x.shape == y.shape
            fake.append(np.asarray(detector(x, return_features=True).cpu(), dtype=np.float32))
            real.append(np.asarray(detector(y, return_features=True).cpu(), dtype=np.float32))
    return np.concatenate(fake), np.concatenate(real)


def mean_cov(rows):
    """Per-row fp64 running sums, then the mean and the /n covariance."""
    s1 = np.zeros(rows.shape[1])
    s2 = np.zeros((rows.shape[1], rows.shape[1]))
    for r in rows.astype(np.float64):
        s1 += r
        s2 += np.outer(r, r)
    mu = s1 / len(rows)
    return mu, s2 / len(rows) - np.outer(mu, mu)


def scores(fake, real):
    mu1, s1 = mean_cov(fake)
    mu2, s2 = mean_cov(real)
    root = scipy.linalg.sqrtm(s1.dot(s2))
    fid = float(np.real(np.square(mu1 - mu2).sum() + np.trace(s1 + s2 - 2 * root)))
    svm = sklearn.svm.LinearSVC(dual=False)
    x = np.concatenate([real, fake])
    t = np.array([1] * len(real) + [0] * len(fake))
    svm.fit(x, t)
    uids = 1 - svm.score(x, t)
    pids = np.mean(svm.decision_function(fake) > svm.decision_function(real))
    return fid, float(pids), float(uids)


def inpainting_metrics(gen_dir, gt_dir, detector, device="cpu"):
    return scores(*features(gen_dir, gt_dir, detector, device))
