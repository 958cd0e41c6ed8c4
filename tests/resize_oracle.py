"""A float64 restatement of Pillow's 8-bit BICUBIC resample, written as Pillow's loops are (one output index, one tap at a
time), independently of gms_b200/dataset.py's vectorised tables: precompute_coeffs + normalize_coeffs_8bpc, then the
horizontal pass over the source rows the vertical pass reads, an 8-bit intermediate, and the vertical pass."""
import math

import numpy as np


def _filter(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size: int, out_size: int):
    """-> (bounds [(xmin, n)], fixed-point weights [out][ksize] as Python ints, ksize)."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds, kk = [], []
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [_filter((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        k += [0.0] * (ksize - xmax)
        kk.append([int(-0.5 + w * (1 << 22)) if w < 0 else int(0.5 + w * (1 << 22)) for w in k])
        bounds.append((xmin, xmax))
    return bounds, kk, ksize


def _pass(img: np.ndarray, bounds, kk, axis: int) -> np.ndarray:
    """One pass along `axis` (1: horizontal, 0: vertical) over uint8 [H,W,C], integer arithmetic."""
    src = img.astype(np.int64)
    out_n = len(bounds)
    shape = list(img.shape)
    shape[axis] = out_n
    out = np.empty(shape, np.uint8)
    for i, (xmin, n) in enumerate(bounds):
        k = np.array(kk[i][:n], np.int64)
        taps = src[:, xmin:xmin + n] if axis == 1 else src[xmin:xmin + n]
        s = (1 << 21) + np.tensordot(taps, k, axes=([axis], [0]))
        assert np.abs(s).max() < 2 ** 31     # Pillow's int32 accumulator does not overflow
        v = np.clip(s >> 22, 0, 255).astype(np.uint8)
        if axis == 1:
            out[:, i] = v
        else:
            out[i] = v
    return out


def resize(img: np.ndarray, width: int, height: int) -> np.ndarray:
    """uint8 [H,W,C] -> [height,width,C] as Image.resize((width, height)) with its default filter."""
    H, W = img.shape[:2]
    horiz, vert = width != W, height != H
    if not horiz and not vert:
        return img.copy()
    bv, kv, _ = coeffs(H, height)
    if horiz:
        bh, kh, _ = coeffs(W, width)
        if vert:
            first, last = bv[0][0], bv[-1][0] + bv[-1][1]
            img = _pass(img[first:last], bh, kh, 1)
            bv = [(x - first, n) for x, n in bv]
        else:
            img = _pass(img, bh, kh, 1)
    if vert:
        img = _pass(img, bv, kv, 0)
    return img


def composite(rgba: np.ndarray, white: bool) -> np.ndarray:
    """readCamerasFromTransforms' numpy sequence (scene/dataset_readers.py:204-210), read back as bytes."""
    norm = rgba / 255.0
    bg = np.array([1, 1, 1]) if white else np.array([0, 0, 0])
    arr = norm[:, :, :3] * norm[:, :, 3:4] + bg * (1 - norm[:, :, 3:4])
    return np.array(arr * 255.0, dtype=np.byte).view(np.uint8)
