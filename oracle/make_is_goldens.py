"""Record tests/golden/is_ref.npz from the UNMODIFIED reference ``pytorch_fid`` package.  Build-container only.

Run:  python oracle/make_is_goldens.py [--check]      (needs /root/reference; never run on the GPU box)

What it pins (tests/test_inception_score_host.py compares ``lfm_b200.fid`` / ``lfm_b200.inception_score`` with it):

* ``logits``: the ``[2, 1008]`` class logits of the reference's own network, ``pytorch_fid.inception.fid_inception_v3()``
  (torchvision ``Inception3`` with the patched blocks and its ``fc``), with the weight download replaced by the seeded
  trunk + ``fc`` dictionary ``synthetic_inception_state_dict(1) | synthetic_fc_state_dict(1)``, on the seeded
  ``[2, 3, 299, 299]`` input in [-1, 1] of :func:`seeded_inputs` (rebuilt by the tests, not stored).
* ``probs_{N}`` and ``mean_{N}_{S}`` / ``std_{N}_{S}``: ``preds2score`` of ``pytorch_fid/inception_score.py`` on seeded
  fp32 probability arrays of N = 37 and 100 rows, S = 1, 3 and 10 splits.  The module is imported with
  ``tensorflow``, ``tensorflow_gan`` and ``tensorflow.python.ops.array_ops`` stubbed by ``MagicMock`` in ``sys.modules``
  (its import-time graph building then touches only the stubs); ``preds2score`` itself is numpy.

TF1's legacy bilinear resize is TensorFlow code, not reference code: tests/tools/inception_score_oracle.py restates it.
"""
import os
import sys
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("LFM_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "is_ref.npz")
SIZES, SPLITS = (37, 100), (1, 3, 10)


def seeded_inputs():
    g = torch.Generator().manual_seed(11)
    return torch.rand(2, 3, 299, 299, generator=g) * 2 - 1


def seeded_probs(n, seed=5):
    rng = np.random.RandomState(seed + n)
    logits = rng.randn(n, 1000) * 2.0 + rng.randn(1, 1000)          # a shared class preference plus per-image noise
    p = np.exp(logits - logits.max(1, keepdims=True))
    return (p / p.sum(1, keepdims=True)).astype(np.float32)


def record():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    from lfm_b200.fid import synthetic_fc_state_dict, synthetic_inception_state_dict
    from pytorch_fid import inception

    sd = {**synthetic_inception_state_dict(1), **synthetic_fc_state_dict(1)}
    inception.load_state_dict_from_url = lambda *a, **k: full
    torch.manual_seed(0)
    full = inception._inception_v3(num_classes=1008, aux_logits=False, weights=None).state_dict()
    for k, v in full.items():          # num_batches_tracked: present in the published file, unused in eval mode
        full[k] = sd.get(k, torch.zeros_like(v))
    net = inception.fid_inception_v3().eval()
    with torch.no_grad():
        logits = net(seeded_inputs())

    stubs = {m: mock.MagicMock() for m in ("tensorflow", "tensorflow.compat", "tensorflow.compat.v1", "tensorflow_gan",
                                           "tensorflow.python", "tensorflow.python.ops", "tensorflow.python.ops.array_ops")}
    with mock.patch.dict(sys.modules, stubs):
        from pytorch_fid import inception_score
    rec = dict(logits=logits.numpy())
    for n in SIZES:
        p = seeded_probs(n)
        rec[f"probs_{n}"] = p
        for s in SPLITS:
            m, sd_ = inception_score.preds2score(p, s)
            rec[f"mean_{n}_{s}"], rec[f"std_{n}_{s}"] = np.float64(m), np.float64(sd_)
    return rec


def main():
    rec = record()
    if "--check" in sys.argv:
        z = np.load(OUT)
        ok = sorted(z.files) == sorted(rec)
        for k in rec:
            same = ok and np.allclose(z[k], rec[k], rtol=1e-6, atol=1e-7)
            print(f"{k}: {'same' if same else 'DIFFERENT'}")
            ok &= bool(same)
        return 0 if ok else 1
    np.savez(OUT, **rec)
    print("wrote", OUT, {k: np.asarray(v).shape for k, v in rec.items()})
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
