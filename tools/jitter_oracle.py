"""CPU restatement of scale-jitter training augmentation (models/pipeline.py RawCollater(scale_jitter=...)), written in
NumPy on top of tools/resize_oracle.py.  tests/test_scale_jitter.py compares the device path (csrc/pipeline.cu
effdet_resize_crop_normalize_pad and effdet_collate_pack_annots_crop) against it; tests/golden/make_jitter_golden.py
pins it to the reference's own Normalizer, Augmenter and Resizer (at common size L) -> tests/golden/pipeline_jitter.npz.

Where the kernel computes each output pixel of the window directly from the source, this oracle takes the long way:
resize the whole image (resize_oracle.resize_linear), zero-pad it to L x L as the Resizer does, and slice the S x S
window at (y0, x0), zero-padded where it runs past the L x L image.

  crop_image    Normalizer -> Augmenter flip -> Resizer at L -> window -> .float(), one image, float32 [3, S, S]
  crop_boxes    the box rule: flip, *= scale, shift by (x0, y0), clamp to [0, S] (fp64), one cast to fp32, drop rows
                whose label is -1 or whose fp32 area is zero
  pack          boxes of a batch -> the [Bcap, Gcap, 5] table (-1 padded) and counts [1 + Bcap]
  from_raw      the same for a RawBatch, from the geometry it recorded (no draws are repeated)
"""
import numpy as np

import resize_oracle as R


def crop_image(img_u8, flip, rh, rw, y0, x0, S, pixel_scale=None):
    """img_u8 uint8 [h, w, 3]; (rh, rw): the Resizer's size at the drawn common size L = max(rh, rw); (y0, x0): the
    window -> float32 [3, S, S]"""
    img = R.normalize(img_u8, pixel_scale)
    if flip:
        img = img[:, ::-1, :]
    L = max(rh, rw)
    full = np.zeros((L, L, 3))                                       # Resizer's new_image at common_size=L
    full[:rh, :rw] = R.resize_linear(img, rh, rw)
    win = full[y0:y0 + S, x0:x0 + S]
    out = np.zeros((S, S, 3))
    out[:win.shape[0], :win.shape[1]] = win
    return out.astype(np.float32).transpose(2, 0, 1)


def _clamp(v, S):
    """v clamped to [0, S]; NaN stays NaN (the kernel's comparisons)"""
    return np.where(v < 0, 0.0, np.where(v > S, float(S), v))


def crop_boxes(rows, flip, width, scale, y0, x0, S):
    """rows float64 [n, 5] (x1, y1, x2, y2, label) of an image of the given width -> the kept rows, float32 [m, 5]"""
    a = np.asarray(rows, dtype=np.float64).reshape(-1, 5).copy()
    if flip:                                                         # Augmenter: cols - x2, cols - x1
        x1, x2 = a[:, 0].copy(), a[:, 2].copy()
        a[:, 0] = float(width) - x2
        a[:, 2] = float(width) - x1
    a[:, :4] *= scale                                                # Resizer
    a[:, [0, 2]] = _clamp(a[:, [0, 2]] - float(x0), S)
    a[:, [1, 3]] = _clamp(a[:, [1, 3]] - float(y0), S)
    f = a.astype(np.float32)
    keep = (f[:, 4] != -1) & (f[:, 2] > f[:, 0]) & (f[:, 3] > f[:, 1])
    return f[keep]


def pack(kept, Bcap, Gcap):
    """kept: per image float32 [m_b, 5] -> (table float32 [Bcap, Gcap, 5], counts int32 [1 + Bcap])"""
    table = np.full((Bcap, Gcap, 5), -1, dtype=np.float32)
    counts = np.zeros(1 + Bcap, dtype=np.int32)
    counts[0] = len(kept)
    for b, k in enumerate(kept):
        table[b, :len(k)] = k
        counts[1 + b] = len(k)
    return table, counts


def from_raw(raw, Gcap, Bcap=None):
    """a scale-jittered RawBatch (host blob) -> (images float32 [Bcap, 3, S, S] with zero padding images, table,
    counts), from the sizes, flips, scales, resized sizes, windows, rows and pixels it recorded"""
    assert raw.jitter
    Bcap = raw.capacity if Bcap is None else Bcap
    S, B = raw.S, raw.B
    a = raw.blob.numpy()
    sec = {n: raw.section(n).numpy() for n in ('offsets', 'hw', 'resized_hw', 'flips', 'scales', 'row_offsets', 'crops')}
    from models.pipeline import raw_layout                           # the blob's format, not its arithmetic
    off, _ = raw_layout(raw.capacity, raw.rows, raw.nbytes, jitter=True)
    rows = a[off['rows']:off['rows'] + 40 * raw.rows].view(np.float64).reshape(-1, 5)
    images = np.zeros((Bcap, 3, S, S), dtype=np.float32)
    kept = []
    for b in range(B):
        h, w = (int(v) for v in sec['hw'][b])
        o = int(sec['offsets'][b])
        img = a[o:o + h * w * 3].reshape(h, w, 3)
        rh, rw = (int(v) for v in sec['resized_hw'][b])
        y0, x0 = (int(v) for v in sec['crops'][b])
        fl = bool(sec['flips'][b])
        images[b] = crop_image(img, fl, rh, rw, y0, x0, S, raw.pixel_scale)
        r = rows[sec['row_offsets'][b]:sec['row_offsets'][b + 1]]
        kept.append(crop_boxes(r, fl, w, float(sec['scales'][b]), y0, x0, S))
    table, counts = pack(kept, Bcap, Gcap)
    return images, table, counts
