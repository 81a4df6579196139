"""FID on the device, fed straight from the decoded uint8 images (SURVEY.md section 8(f)-4).

The reference writes every sample as a JPEG, then ``pytorch_fid`` reads the directory back through a DataLoader, runs
the "FID Inception" network and computes the Frechet distance with numpy / scipy on the host
(/root/reference/pytorch_fid/fid_score.py:114-175 activations, :178-228 distance, :231-283 driver;
/root/reference/pytorch_fid/inception.py:24-163 the network, :182-331 its TensorFlow-compatibility patches).  Here the
images never leave the GPU:

* :class:`FIDInception` is the same network - torchvision ``inception_v3`` layer names, so that the published
  ``pt_inception-2015-12-05`` weight file loads by key - as ONE table of branches interpreted by a small loop, with every
  BatchNorm folded into its convolution when the weights are loaded.  The three TensorFlow quirks the reference patches
  in are table entries: 3x3 average pools that do not count the zero padding (inception.py:201-203, 231-233, 264-266) and
  the max pool in the last block (inception.py:321-326).  It accepts the decoder's ``[B, H, W, 3]`` uint8 batch (or
  ``[B, 3, H, W]`` floats in [0, 1], the reference's input) and returns the ``[B, 2048]`` pool3 features.
  The convolutions themselves are library calls (cuDNN through torch): SURVEY.md 8(f)-4 lists this row as library work;
  what this module removes is the JPEG + host round trip and the host-side statistics.
* :class:`FIDStatistics` keeps the running sum and the running sum of outer products in fp64 on the device; ranks combine
  them with ONE all-reduce (no feature gather); ``finalize`` gives the mean and the unbiased covariance
  (``np.mean`` / ``np.cov(rowvar=False)``, fid_score.py:224-226).
* :func:`frechet_distance` evaluates ``|mu1 - mu2|^2 + Tr(S1) + Tr(S2) - 2 Tr(sqrt(S1 S2))`` (fid_score.py:178-228)
  through two symmetric eigen-decompositions in fp64: ``Tr sqrt(S1 S2) = sum sqrt(eig(S1^1/2 S2 S1^1/2))``, the same
  number ``scipy.linalg.sqrtm`` gives whenever its result is real, without the complex Schur form and on the GPU.
* :func:`load_statistics` reads the reference's ``*_stat.npy`` / ``.npz`` files (fid_score.py:231-238).
* ``python -m lfm_b200.fid PATH PATH --inception_weights FILE`` is ``pytorch_fid/fid_score.py PATH PATH``: FID between two
  image directories and / or statistics files (fid_score.py:254-295), through the classes above.

Note on parity with a reference run: the reference's number is computed from JPEG-compressed files (quality 75 by PIL's
default); feeding the uint8 images directly removes that compression from the statistic.  ``test_flow_latent.py
--compute_fid`` still writes the files, so ``pytorch_fid`` can be run on them for the number with the compression in it.
"""
from __future__ import annotations

import argparse
import os
import pathlib
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------------------------------------------------
# the network, as data.  conv(name, cin, cout, kernel, stride, padding); every conv is conv -> BN(eps 1e-3) -> ReLU
# (torchvision BasicConv2d, which inception.py:166-179 instantiates).  Kernel / padding are (h, w).
# ---------------------------------------------------------------------------------------------------------------------
_BN_EPS = 1e-3


def _c(name, cin, cout, k=1, s=1, p=0):
    k = (k, k) if isinstance(k, int) else k
    p = (p, p) if isinstance(p, int) else p
    return ("conv", name, cin, cout, k, s, p)


_STEM = [
    _c("Conv2d_1a_3x3", 3, 32, 3, 2), _c("Conv2d_2a_3x3", 32, 32, 3), _c("Conv2d_2b_3x3", 32, 64, 3, 1, 1), ("maxpool",),
    _c("Conv2d_3b_1x1", 64, 80), _c("Conv2d_4a_3x3", 80, 192, 3), ("maxpool",),
]


def _block_a(cin, pool_features):
    return [
        [_c("branch1x1", cin, 64)],
        [_c("branch5x5_1", cin, 48), _c("branch5x5_2", 48, 64, 5, 1, 2)],
        [_c("branch3x3dbl_1", cin, 64), _c("branch3x3dbl_2", 64, 96, 3, 1, 1), _c("branch3x3dbl_3", 96, 96, 3, 1, 1)],
        [("avgpool_nopad",), _c("branch_pool", cin, pool_features)],
    ]


def _block_b(cin):
    return [
        [_c("branch3x3", cin, 384, 3, 2)],
        [_c("branch3x3dbl_1", cin, 64), _c("branch3x3dbl_2", 64, 96, 3, 1, 1), _c("branch3x3dbl_3", 96, 96, 3, 2)],
        [("maxpool",)],
    ]


def _block_c(cin, c7):
    row, col = (1, 7), (7, 1)
    prow, pcol = (0, 3), (3, 0)
    return [
        [_c("branch1x1", cin, 192)],
        [_c("branch7x7_1", cin, c7), _c("branch7x7_2", c7, c7, row, 1, prow), _c("branch7x7_3", c7, 192, col, 1, pcol)],
        [_c("branch7x7dbl_1", cin, c7), _c("branch7x7dbl_2", c7, c7, col, 1, pcol), _c("branch7x7dbl_3", c7, c7, row, 1, prow),
         _c("branch7x7dbl_4", c7, c7, col, 1, pcol), _c("branch7x7dbl_5", c7, 192, row, 1, prow)],
        [("avgpool_nopad",), _c("branch_pool", cin, 192)],
    ]


def _block_d(cin):
    return [
        [_c("branch3x3_1", cin, 192), _c("branch3x3_2", 192, 320, 3, 2)],
        [_c("branch7x7x3_1", cin, 192), _c("branch7x7x3_2", 192, 192, (1, 7), 1, (0, 3)),
         _c("branch7x7x3_3", 192, 192, (7, 1), 1, (3, 0)), _c("branch7x7x3_4", 192, 192, 3, 2)],
        [("maxpool",)],
    ]


def _block_e(cin, pool):
    # a branch entry ("fork", [convs...]) applies each conv to the same input and concatenates (the 1x3 / 3x1 pairs)
    return [
        [_c("branch1x1", cin, 320)],
        [_c("branch3x3_1", cin, 384),
         ("fork", [_c("branch3x3_2a", 384, 384, (1, 3), 1, (0, 1)), _c("branch3x3_2b", 384, 384, (3, 1), 1, (1, 0))])],
        [_c("branch3x3dbl_1", cin, 448), _c("branch3x3dbl_2", 448, 384, 3, 1, 1),
         ("fork", [_c("branch3x3dbl_3a", 384, 384, (1, 3), 1, (0, 1)), _c("branch3x3dbl_3b", 384, 384, (3, 1), 1, (1, 0))])],
        [(pool,), _c("branch_pool", cin, 192)],
    ]


_MIXED = [
    ("Mixed_5b", _block_a(192, 32)), ("Mixed_5c", _block_a(256, 64)), ("Mixed_5d", _block_a(288, 64)),
    ("Mixed_6a", _block_b(288)),
    ("Mixed_6b", _block_c(768, 128)), ("Mixed_6c", _block_c(768, 160)), ("Mixed_6d", _block_c(768, 160)),
    ("Mixed_6e", _block_c(768, 192)),
    ("Mixed_7a", _block_d(768)),
    ("Mixed_7b", _block_e(1280, "avgpool_nopad")),   # inception.py:262-266
    ("Mixed_7c", _block_e(2048, "maxpool_same")),    # inception.py:321-326: the FID graph max-pools here
]


def _all_convs():
    for op in _STEM:
        if op[0] == "conv":
            yield op[1], op
    for block, branches in _MIXED:
        for branch in branches:
            for op in branch:
                if op[0] == "conv":
                    yield f"{block}.{op[1]}", op
                elif op[0] == "fork":
                    for sub in op[1]:
                        yield f"{block}.{sub[1]}", sub


def inception_state_dict_shapes() -> Dict[str, Tuple[int, ...]]:
    """Key -> shape of the tensors :meth:`FIDInception.load_state_dict_folded` consumes (the torchvision names the
    published weight file uses; its ``num_batches_tracked`` entries are ignored, and its ``fc.*`` entries are read only by
    a network built ``with_logits``, see :data:`FC_SHAPES`)."""
    out = {}
    for name, (_, _, cin, cout, k, _, _) in _all_convs():
        out[f"{name}.conv.weight"] = (cout, cin, k[0], k[1])
        for leaf in ("weight", "bias", "running_mean", "running_var"):
            out[f"{name}.bn.{leaf}"] = (cout,)
    return out


FC_SHAPES = {"fc.weight": (1008, 2048), "fc.bias": (1008,)}   # the graph's softmax/logits layer: 1008 classes


def _keyed_generator(seed: int, key: str) -> torch.Generator:
    import zlib
    return torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(key.encode())) % (2 ** 31))


def synthetic_inception_state_dict(seed: int = 1) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for the published weights (there is no network here): He-scaled convolutions and BatchNorm
    statistics near the identity, every tensor drawn from a generator keyed on (seed, crc32(key)) so that the
    reference-side fixture script and the tests build the identical dictionary without shipping 95 MB."""
    sd = {}
    for key, shape in inception_state_dict_shapes().items():
        g = _keyed_generator(seed, key)
        if key.endswith("conv.weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif key.endswith("running_var") or key.endswith("bn.weight"):
            t = 0.8 + 0.4 * torch.rand(shape, generator=g)
        else:
            t = 0.05 * torch.randn(shape, generator=g)
        sd[key] = t
    return sd


def synthetic_fc_state_dict(seed: int = 1) -> Dict[str, torch.Tensor]:
    """Seeded stand-in for the ``fc.*`` classifier of the published file, keyed as :func:`synthetic_inception_state_dict`
    is: a weight of std ``4 / sqrt(2048)`` (logits of a few units, so the softmax is neither flat nor one-hot on the
    stand-in trunk's features) and a bias of std 0.05."""
    sd = {}
    for key, shape in FC_SHAPES.items():
        g = _keyed_generator(seed, key)
        sd[key] = torch.randn(shape, generator=g) * (4.0 / 2048 ** 0.5 if key == "fc.weight" else 0.05)
    return sd


class FIDInception(torch.nn.Module):
    """pool3 (2048-d) features of the FID Inception graph; see the module docstring.  With ``with_logits`` it also holds
    the graph's ``fc`` layer (``fc.weight [1008, 2048]``, ``fc.bias [1008]`` of the same weight file, loaded strictly)
    and :meth:`logits` gives the 1008 class logits the Inception Score uses (lfm_b200/inception_score.py)."""

    def __init__(self, state_dict: Optional[Dict[str, torch.Tensor]] = None, allow_tf32: bool = False,
                 with_logits: bool = False):
        super().__init__()
        self.allow_tf32 = bool(allow_tf32)
        self.with_logits = bool(with_logits)
        self._loaded = False
        for name, (_, _, cin, cout, k, _, _) in _all_convs():
            self.register_buffer(self._w(name), torch.zeros(cout, cin, k[0], k[1]), persistent=False)
            self.register_buffer(self._b(name), torch.zeros(cout), persistent=False)
        if self.with_logits:
            self.register_buffer("fc_w", torch.zeros(FC_SHAPES["fc.weight"]), persistent=False)
            self.register_buffer("fc_b", torch.zeros(FC_SHAPES["fc.bias"]), persistent=False)
        if state_dict is not None:
            self.load_state_dict_folded(state_dict)

    @staticmethod
    def _w(name):
        return "w_" + name.replace(".", "__")

    @staticmethod
    def _b(name):
        return "b_" + name.replace(".", "__")

    @classmethod
    def from_file(cls, path: str, **kw) -> "FIDInception":
        """``path``: a local copy of ``pt_inception-2015-12-05-6726825d.pth`` (inception.py:20; no download here)."""
        if not os.path.isfile(path):
            raise FileNotFoundError(f"Inception weight file not found: {path} (there is no network access; pass a local "
                                    "copy of pt_inception-2015-12-05-6726825d.pth)")
        return cls(torch.load(path, map_location="cpu", weights_only=True), **kw)

    @torch.no_grad()
    def load_state_dict_folded(self, sd: Dict[str, torch.Tensor]) -> None:
        """Folds BN(eps 1e-3, eval mode) into each convolution in fp64: w' = w * g / sqrt(var + eps),
        b' = beta - mean * g / sqrt(var + eps).  Raises KeyError / ValueError on a missing or mis-shaped tensor.  The
        ``fc.*`` entries are read only by a network built ``with_logits``; it raises ValueError when they are missing."""
        shapes = inception_state_dict_shapes()
        missing = [k for k in shapes if k not in sd]
        if missing:
            raise KeyError(f"Inception state dict lacks {len(missing)} tensors, e.g. {missing[:3]}")
        if self.with_logits:
            missing = [k for k in FC_SHAPES if k not in sd]
            if missing:
                raise ValueError(f"Inception state dict lacks {missing}: the class logits need the graph's fc layer "
                                 "(pt_inception-2015-12-05-6726825d.pth has it)")
            shapes = {**shapes, **FC_SHAPES}
        for k, shp in shapes.items():
            if tuple(sd[k].shape) != shp:
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)}, expected {shp}")
        for name, _ in _all_convs():
            w = sd[f"{name}.conv.weight"].double()
            g = sd[f"{name}.bn.weight"].double() / torch.sqrt(sd[f"{name}.bn.running_var"].double() + _BN_EPS)
            b = sd[f"{name}.bn.bias"].double() - sd[f"{name}.bn.running_mean"].double() * g
            getattr(self, self._w(name)).copy_((w * g[:, None, None, None]).float())
            getattr(self, self._b(name)).copy_(b.float())
        if self.with_logits:
            self.fc_w.copy_(sd["fc.weight"].float())
            self.fc_b.copy_(sd["fc.bias"].float())
        self._loaded = True

    # -- interpreter ---------------------------------------------------------------------------------------------------
    def _conv(self, x, prefix, op):
        _, name, _, _, _, s, p = op
        full = prefix + name
        return F.relu_(F.conv2d(x, getattr(self, self._w(full)), getattr(self, self._b(full)), stride=s, padding=p))

    def _run(self, x, prefix, ops):
        for op in ops:
            kind = op[0]
            if kind == "conv":
                x = self._conv(x, prefix, op)
            elif kind == "maxpool":
                x = F.max_pool2d(x, 3, 2)
            elif kind == "maxpool_same":
                x = F.max_pool2d(x, 3, 1, 1)
            elif kind == "avgpool_nopad":
                x = F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)
            elif kind == "fork":
                x = torch.cat([self._conv(x, prefix, sub) for sub in op[1]], 1)
            else:
                raise AssertionError(kind)
        return x

    @staticmethod
    def prepare(images: torch.Tensor) -> torch.Tensor:
        """uint8 ``[B, H, W, 3]`` (the decoder's output) or float ``[B, 3, H, W]`` in [0, 1] -> ``[B, 3, 299, 299]`` in
        [-1, 1]: ToTensor's /255 (fid_score.py:147), bilinear resize without corner alignment, 2x - 1 (inception.py:153-157)."""
        if images.dtype == torch.uint8:
            if images.dim() != 4 or images.shape[-1] != 3:
                raise ValueError(f"uint8 images must be [B, H, W, 3], got {tuple(images.shape)}")
            x = images.permute(0, 3, 1, 2).float() / 255.0
        else:
            if images.dim() != 4 or images.shape[1] != 3:
                raise ValueError(f"float images must be [B, 3, H, W], got {tuple(images.shape)}")
            x = images.float()
        x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
        return 2 * x - 1

    @torch.no_grad()
    def forward(self, images: torch.Tensor) -> torch.Tensor:
        return self.trunk(self.prepare(images))

    @torch.no_grad()
    def trunk(self, x: torch.Tensor) -> torch.Tensor:
        """Prepared ``[B, 3, 299, 299]`` input in [-1, 1] -> ``[B, 2048]`` pool3 features."""
        if not self._loaded:
            raise RuntimeError("FIDInception has no weights: load_state_dict_folded / from_file first")
        cudnn_tf32 = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = self.allow_tf32
        try:
            if x.is_cuda:
                x = x.contiguous(memory_format=torch.channels_last)
            x = self._run(x, "", _STEM)
            for block, branches in _MIXED:
                x = torch.cat([self._run(x, block + ".", br) for br in branches], 1)
            return x.mean(dim=(2, 3))
        finally:
            torch.backends.cudnn.allow_tf32 = cudnn_tf32

    @torch.no_grad()
    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """Prepared ``[B, 3, 299, 299]`` input in [-1, 1] -> ``[B, 1008]`` logits: the trunk, then ``fc`` in fp32
        (the graph's ``softmax/logits``)."""
        if not self.with_logits:
            raise RuntimeError("FIDInception was built without its fc layer: pass with_logits=True")
        matmul_tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = self.allow_tf32
        try:
            return F.linear(self.trunk(x), self.fc_w, self.fc_b)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = matmul_tf32


# ---------------------------------------------------------------------------------------------------------------------
# statistics and distance
# ---------------------------------------------------------------------------------------------------------------------
class FIDStatistics:
    """Running mean / covariance of feature rows, fp64 on the device of the first update."""

    def __init__(self, dims: int = 2048, device=None):
        self.dims = dims
        self.n = 0
        self.s1 = torch.zeros(dims, dtype=torch.float64, device=device)
        self.s2 = torch.zeros(dims, dims, dtype=torch.float64, device=device)

    def update(self, feats: torch.Tensor) -> None:
        if feats.dim() != 2 or feats.shape[1] != self.dims:
            raise ValueError(f"features must be [B, {self.dims}], got {tuple(feats.shape)}")
        if self.s1.device != feats.device:
            self.s1, self.s2 = self.s1.to(feats.device), self.s2.to(feats.device)
        f = feats.double()
        self.n += f.shape[0]
        self.s1 += f.sum(0)
        self.s2 += f.t() @ f

    def all_reduce(self) -> None:
        """Sum over the ranks of the default process group: one collective on a [dims + 1, dims] buffer plus the count."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return
        buf = torch.cat([self.s2, self.s1[None, :]], 0)
        cnt = torch.tensor([float(self.n)], dtype=torch.float64, device=buf.device)
        dist.all_reduce(buf)
        dist.all_reduce(cnt)
        self.s2, self.s1, self.n = buf[:-1].clone(), buf[-1].clone(), int(round(cnt.item()))

    def finalize(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """(mu [dims], sigma [dims, dims]) with the N-1 normalisation of ``np.cov`` (fid_score.py:225)."""
        if self.n < 2:
            raise ValueError("at least two feature rows are needed for a covariance")
        mu = self.s1 / self.n
        sigma = (self.s2 - self.n * torch.outer(mu, mu)) / (self.n - 1)
        return mu, 0.5 * (sigma + sigma.t())


def _as_f64(x, device):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(np.ascontiguousarray(x))
    return x.to(device=device, dtype=torch.float64)


def _sqrt_psd(m: torch.Tensor) -> torch.Tensor:
    w, v = torch.linalg.eigh(m)
    return (v * w.clamp_min(0).sqrt()) @ v.t()


def frechet_distance(mu1, sigma1, mu2, sigma2, device=None) -> float:
    """fid_score.py:178-228 for symmetric positive semi-definite covariances (which sample covariances are).
    Negative eigenvalues from round-off are clamped to zero, the counterpart of the reference dropping the imaginary
    part of ``sqrtm`` (fid_score.py:214-219)."""
    if device is None:
        device = mu1.device if isinstance(mu1, torch.Tensor) else torch.device("cpu")
    mu1, mu2 = _as_f64(mu1, device).reshape(-1), _as_f64(mu2, device).reshape(-1)
    s1, s2 = _as_f64(sigma1, device), _as_f64(sigma2, device)
    if s1.dim() < 2:
        s1, s2 = s1.reshape(1, 1), s2.reshape(1, 1)
    if mu1.shape != mu2.shape:
        raise ValueError("Training and test mean vectors have different lengths")
    if s1.shape != s2.shape:
        raise ValueError("Training and test covariances have different dimensions")
    s1, s2 = 0.5 * (s1 + s1.t()), 0.5 * (s2 + s2.t())
    a = _sqrt_psd(s1)
    m = a @ s2 @ a
    tr_covmean = torch.linalg.eigvalsh(0.5 * (m + m.t())).clamp_min(0).sqrt().sum()
    diff = mu1 - mu2
    return float(diff @ diff + torch.trace(s1) + torch.trace(s2) - 2 * tr_covmean)


def load_statistics(path: str) -> Tuple[np.ndarray, np.ndarray]:
    """The reference's precomputed dataset statistics: ``.npz`` with mu / sigma arrays, or ``.npy`` holding a pickled
    dict (fid_score.py:231-238; e.g. pytorch_fid/celebahq_stat.npy)."""
    f = np.load(path, allow_pickle=True)
    if isinstance(f, np.lib.npyio.NpzFile):
        return np.asarray(f["mu"]), np.asarray(f["sigma"])
    d = f.item() if f.dtype == object else f
    return np.asarray(d["mu"]), np.asarray(d["sigma"])


class FIDAccumulator:
    """What the generation loop holds: network + statistics.  ``update(images_uint8_nhwc)`` per batch on each rank,
    ``compute(real_stats_path)`` once at the end (collective when a process group is up; every rank gets the number)."""

    def __init__(self, net: FIDInception, device, batch: int = 200):
        self.net = net.to(device)
        self.stats = FIDStatistics(2048, device)
        self.batch = batch   # fid_score.py:271 batch_size=200 from test_flow_latent.py:277

    def update(self, images: torch.Tensor) -> None:
        for i in range(0, images.shape[0], self.batch):
            self.stats.update(self.net(images[i:i + self.batch]))

    def compute(self, real_stats_path: str) -> float:
        self.stats.all_reduce()
        mu, sigma = self.stats.finalize()
        m2, s2 = load_statistics(real_stats_path)
        return frechet_distance(mu, sigma, m2, s2, device=mu.device)


# ---------------------------------------------------------------------------------------------------------------------
# FID between two paths (pytorch_fid/fid_score.py:254-295)
# ---------------------------------------------------------------------------------------------------------------------
IMAGE_EXTENSIONS = {"bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp"}   # fid_score.py:95


def list_images(path: str):
    """The images of a directory as fid_score.py:263 takes them: its files (not its subdirectories') with an extension of
    IMAGE_EXTENSIONS, sorted."""
    root = pathlib.Path(path)
    return sorted(f for ext in IMAGE_EXTENSIONS for f in root.glob("*.{}".format(ext)))


def statistics_of_path(path: str, net: FIDInception, batch_size: int = 50, device=None) -> Tuple[np.ndarray, np.ndarray]:
    """fid_score.py:254-265: ``.npz`` / ``.npy`` statistics are read; a directory's images, converted to RGB, go through the
    network as uint8 batches of ``batch_size`` and are summed by :class:`FIDStatistics`.  The images of a batch must share
    one size, as the reference's DataLoader collate requires."""
    from PIL import Image
    if path.endswith(".npz") or path.endswith(".npy"):
        return load_statistics(path)
    if batch_size < 1:
        raise ValueError(f"batch size must be >= 1, got {batch_size}")
    stats = FIDStatistics(2048, device)
    files = list_images(path)
    for i in range(0, len(files), batch_size):
        batch = [np.asarray(Image.open(f).convert("RGB")) for f in files[i:i + batch_size]]
        sizes = sorted({b.shape for b in batch})
        if len(sizes) > 1:
            raise ValueError(f"{path}: images of one batch differ in size ({', '.join(f'{h}x{w}' for h, w, _ in sizes)}), "
                             f"from {files[i].name}")
        stats.update(net(torch.from_numpy(np.stack(batch)).to(device)))
    mu, sigma = stats.finalize()
    return mu.cpu().numpy(), sigma.cpu().numpy()


def build_parser():
    p = argparse.ArgumentParser("python -m lfm_b200.fid", description="FID between two image directories or statistics files")
    p.add_argument("path", type=str, nargs=2, help="paths to the generated images or to .npz / .npy statistics files")
    p.add_argument("--inception_weights", type=str, required=True,
                   help="local copy of pt_inception-2015-12-05-6726825d.pth (there is no download)")
    p.add_argument("--batch-size", type=int, default=50, help="images per network call")
    p.add_argument("--device", type=str, default=None, help="cuda, cuda:N or cpu (default: cuda when available)")
    p.add_argument("--dims", type=int, default=2048, choices=[2048], help="pool3 features (the only ones computed here)")
    return p


def main(argv=None) -> float:
    args = build_parser().parse_args(argv)
    for p in args.path:
        if not os.path.exists(p):
            raise RuntimeError("Invalid path: %s" % p)
    device = torch.device(args.device if args.device else ("cuda" if torch.cuda.is_available() else "cpu"))
    net = FIDInception.from_file(args.inception_weights).to(device).eval()
    m1, s1 = statistics_of_path(args.path[0], net, args.batch_size, device)
    m2, s2 = statistics_of_path(args.path[1], net, args.batch_size, device)
    value = frechet_distance(m1, s1, m2, s2, device=device)
    print("FID: ", value)
    return value


if __name__ == "__main__":
    main()
