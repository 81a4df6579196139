"""numpy restatement of the input pipeline of ``pytorch_fid/inception_score.py`` (:50-52, :74): ``x / 255 * 2 - 1`` in
float64 (numpy promotes the array), fp32 from there on, NCHW -> NHWC, then ``tf.compat.v1.image.resize_bilinear`` to
299 x 299.

The resize is TensorFlow's kernel, not reference code, and TensorFlow is not available to pin it: this is restated from
memory of TF's ``resize_bilinear_op.cc`` with ``align_corners=False, half_pixel_centers=False`` (the TF1 defaults), and
is unpinned.  Per output axis, in fp32: ``scale = in / out``, ``src = dst * scale``, ``lower = floor(src)``,
``upper = min(ceil(src), in - 1)``, ``lerp = src - floor(src)``; a pixel is ``top + (bottom - top) * y_lerp`` with
``top = top_left + (top_right - top_left) * x_lerp`` (and ``bottom`` alike).
"""
import numpy as np


def _axis(n_in, n_out):
    scale = np.float32(n_in) / np.float32(n_out)
    src = np.arange(n_out, dtype=np.float32) * scale
    lower = np.maximum(np.floor(src).astype(np.int64), 0)
    upper = np.minimum(np.ceil(src).astype(np.int64), n_in - 1)
    return lower, upper, (src - np.floor(src)).astype(np.float32)


def resize_bilinear_tf1(x_nhwc, size=299):
    """``[B, H, W, C]`` fp32 -> ``[B, size, size, C]`` fp32."""
    x = np.asarray(x_nhwc, dtype=np.float32)
    yl, yu, ly = _axis(x.shape[1], size)
    xl, xu, lx = _axis(x.shape[2], size)
    lx = lx[None, None, :, None]

    def across(rows):
        left, right = rows[:, :, xl], rows[:, :, xu]
        return left + (right - left) * lx
    top, bottom = across(x[:, yl]), across(x[:, yu])
    return top + (bottom - top) * ly[None, :, None, None]


def prepare_reference(images_nchw):
    """``[B, 3, H, W]`` values in 0..255 -> the network input ``[B, 3, 299, 299]`` fp32 (NCHW, for comparison)."""
    inp = (np.asarray(images_nchw) / 255.0 * 2 - 1).astype(np.float32)
    return resize_bilinear_tf1(inp.transpose(0, 2, 3, 1)).transpose(0, 3, 1, 2)
