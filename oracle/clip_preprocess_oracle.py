"""CPU restatement of the image pre-processing step that feeds the hot path (SURVEY.md §8(f) row 3).

TEST INFRASTRUCTURE ONLY — like everything under oracle/, this file is the checker: only tests/, __graft_entry__.smoke()
and bench.py's CPU legs may import it.  The product never does.

What it restates
  The reference turns a PIL image into `pixel_values` with HF's CLIPImageProcessor
  (models/visualcla/modeling_utils.py:130 builds it, :150/:152/:187/:189 call it); in the reference's pinned
  transformers (4.x) that is the PIL/numpy pipeline of HF:models/clip/image_processing_clip.py:22-33
      convert RGB -> resize(shortest_edge=224, BICUBIC) -> center_crop(224,224) -> rescale(1/255) -> normalize(mean,std)
  whose only non-trivial arithmetic lives in a third-party dependency that is not vendored in the reference:
  Pillow's `ImagingResample` (src/libImaging/Resample.c; behaviour unchanged across Pillow 7 … 12).  Its published
  algorithm for 8-bit images is restated below in integer numpy: separable, antialiased (filter support scaled by the
  down-scaling factor), coefficients quantised to 22 fractional bits, a rounding shift and an 8-bit clip after EACH pass,
  horizontal pass first.  Everything is integer until the final rescale/normalise, so the bar is bit-exact.

Pinned by oracle/gen_golden_preprocess.py against (1) PIL.Image.resize itself and (2) transformers' PIL-backed
CLIPImageProcessor, both run in the build container; the vectors live in tests/golden/preprocess.npz.
"""
import math

import numpy as np

PRECISION_BITS = 32 - 8 - 2            # Pillow Resample.c: PRECISION_BITS
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # HF:utils/constants.py OPENAI_CLIP_MEAN
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)     # HF:utils/constants.py OPENAI_CLIP_STD


def bicubic_weight(x: float) -> float:
    """Pillow Resample.c bicubic_filter (Keys kernel, a = -0.5), support 2."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def resample_coeffs(in_size: int, out_size: int):
    """Pillow Resample.c precompute_coeffs + normalize_coeffs_8bpc for the full-image box (in0 = 0, in1 = in_size).
    Returns (xmin[out], count[out], k[out, ksize] int32).  All intermediate arithmetic is C `double`."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    xmin = np.zeros(out_size, np.int32)
    cnt = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    inv = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        lo = int(center - support + 0.5)            # C (int) cast: truncation toward zero
        lo = max(lo, 0)
        hi = int(center + support + 0.5)
        hi = min(hi, in_size)
        n = hi - lo
        w = [bicubic_weight((x + lo - center + 0.5) * inv) for x in range(n)]
        ww = 0.0
        for v in w:                                  # same left-to-right accumulation order as the C loop
            ww += v
        for x in range(n):
            v = w[x] / ww if ww != 0.0 else w[x]
            v = v * (1 << PRECISION_BITS)
            kk[xx, x] = int(-0.5 + v) if v < 0 else int(0.5 + v)
        xmin[xx], cnt[xx] = lo, n
    return xmin, cnt, kk


def _pass_axis0(img: np.ndarray, out_size: int) -> np.ndarray:
    """One resampling pass along axis 0 of a uint8 array (any trailing shape): int32 accumulate from 1<<(P-1),
    arithmetic shift, clip to 0..255 (Pillow's clip8 lookup)."""
    xmin, cnt, kk = resample_coeffs(img.shape[0], out_size)
    out = np.empty((out_size,) + img.shape[1:], np.uint8)
    src = img.astype(np.int64)
    for xx in range(out_size):
        n = int(cnt[xx])
        seg = src[xmin[xx]:xmin[xx] + n]
        k = kk[xx, :n].astype(np.int64).reshape((n,) + (1,) * (img.ndim - 1))
        acc = (seg * k).sum(axis=0) + (1 << (PRECISION_BITS - 1))
        out[xx] = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return out


def resize_bicubic_u8(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """PIL.Image.resize((out_w, out_h), BICUBIC) on an (H, W, C) uint8 image: horizontal pass, then vertical pass over
    its 8-bit result (ImagingResample); a pass whose size does not change is skipped."""
    assert img.dtype == np.uint8 and img.ndim == 3
    h, w, _ = img.shape
    cur = img
    if out_w != w:
        cur = np.ascontiguousarray(np.swapaxes(_pass_axis0(np.swapaxes(cur, 0, 1), out_w), 0, 1))
    if out_h != h:
        cur = _pass_axis0(cur, out_h)
    return cur


def resize_output_size(h: int, w: int, shortest_edge: int = 224):
    """HF:image_transforms.get_resize_output_image_size(size=int, default_to_square=False): the short side becomes
    `shortest_edge`, the long side int(shortest_edge * long / short) (truncation)."""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = shortest_edge, int(shortest_edge * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)          # (out_h, out_w)


def center_crop_box(h: int, w: int, crop: int = 224):
    """HF:image_transforms.center_crop: top = (h - crop)//2, left = (w - crop)//2 (no padding case: both sides >= crop
    always holds after the shortest-edge resize)."""
    return (h - crop) // 2, (w - crop) // 2


def resize_and_crop_u8(img: np.ndarray, size: int = 224) -> np.ndarray:
    oh, ow = resize_output_size(img.shape[0], img.shape[1], size)
    r = resize_bicubic_u8(img, oh, ow)
    top, left = center_crop_box(oh, ow, size)
    return r[top:top + size, left:left + size]


def rescale_normalize(u8_hwc: np.ndarray) -> np.ndarray:
    """HF rescale (uint8 * (1/255) in float64, cast to float32) then normalize ((x - mean) / std in float32); CHW out."""
    x = (u8_hwc.astype(np.float64) * (1 / 255)).astype(np.float32)
    mean = np.asarray(CLIP_MEAN, dtype=np.float32)
    std = np.asarray(CLIP_STD, dtype=np.float32)
    x = (x - mean) / std
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def clip_preprocess(img_u8_hwc: np.ndarray, size: int = 224) -> np.ndarray:
    """RGB uint8 (H, W, 3) -> pixel_values float32 (3, size, size)."""
    return rescale_normalize(resize_and_crop_u8(img_u8_hwc, size))


def synthetic_image(h: int, w: int, seed: int) -> np.ndarray:
    """Deterministic test picture: smooth gradients + hard edges + mild noise (exercises overshoot clipping)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([127 + 120 * np.sin(xx / (7 + seed % 5)) * np.cos(yy / 11),
                     255 * (((xx // 9 + yy // 13) % 2) == 0),
                     255 * xx / max(w - 1, 1) * (yy / max(h - 1, 1))], axis=-1)
    base += rng.integers(-12, 13, size=base.shape)
    return np.clip(base, 0, 255).astype(np.uint8)
