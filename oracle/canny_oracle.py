"""TEST INFRASTRUCTURE — CPU restatement of the Canny control-map front-end (SURVEY.md §8 row f3):
condition/canny.py:14 `cv2.Canny(img, low_threshold, high_threshold)` on an (H, W, 3) uint8 image -> (H, W) uint8 map
of {0, 255}, which the sampling / demo code turns into the control tensor `2 * (map / 255 - 0.5)` repeated over 3 channels.

The arithmetic lives in a third-party dependency, OpenCV (`opencv-python`, unpinned in the reference's requirements.txt; installed
here: 4.13.0).  Published algorithm of `cv::Canny` (aperture 3, L2gradient = false), all integer:
  * Sobel dx, dy per channel, 3x3, BORDER_REPLICATE, 16-bit;  norm = |dx| + |dy|;  per pixel the FIRST channel with the largest norm
    supplies (mag, xs, ys);  the magnitude map has a zero border.
  * non-maximum suppression for mag > low (= floor(low_threshold)), direction by fixed-point tangents (TG22 = round(tan 22.5 * 2^15)):
      |ys| << 15 <  |xs| * TG22               : keep if mag >  left  and mag >= right
      |ys| << 15 >  |xs| * TG22 + (|xs| << 16): keep if mag >  up    and mag >= down
      otherwise (diagonal)                    : keep if mag >  d1    and mag >  d2, the two neighbours along the gradient's diagonal
                                                (up-left / down-right when xs, ys have the same sign, else up-right / down-left)
  * kept pixels with mag > high (= floor(high_threshold)) are edges; kept pixels with mag <= high become edges when 8-connected
    (transitively) to an edge.
Pinned bit-exactly against cv2.Canny itself (tests/test_frontend_cpu.py, when cv2 is importable) and against a committed fixture
made by cv2 4.13.0 (tests/golden/canny.npz, tests/golden/make_golden.py:canny_case)."""
from __future__ import annotations

import numpy as np

TG22 = 13573   # (int)(0.4142135623730950488016887242097 * (1 << 15) + 0.5)


def sobel_replicate(img: np.ndarray):
    p = np.pad(img.astype(np.int32), ((1, 1), (1, 1), (0, 0)), mode="edge")
    dx = (p[:-2, 2:] + 2 * p[1:-1, 2:] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[1:-1, :-2] + p[2:, :-2])
    dy = (p[2:, :-2] + 2 * p[2:, 1:-1] + p[2:, 2:]) - (p[:-2, :-2] + 2 * p[:-2, 1:-1] + p[:-2, 2:])
    return dx, dy


def canny_classes(img: np.ndarray, low_threshold: float = 100, high_threshold: float = 200):
    """-> (strong, weak) boolean maps after non-maximum suppression and the double threshold."""
    if img.ndim == 2:
        img = img[:, :, None]
    H, W, _ = img.shape
    dx, dy = sobel_replicate(img)
    norm = np.abs(dx) + np.abs(dy)
    idx = np.argmax(norm, axis=2)                       # first channel with the largest norm
    ii, jj = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    m, xs, ys = norm[ii, jj, idx], dx[ii, jj, idx], dy[ii, jj, idx]
    low, high = int(np.floor(min(low_threshold, high_threshold))), int(np.floor(max(low_threshold, high_threshold)))
    mp = np.pad(m, 1)                                   # zero border
    x, y = np.abs(xs), np.abs(ys) << 15
    tg22x = x * TG22
    tg67x = tg22x + (x << 16)
    left, right, up, down = mp[1:-1, :-2], mp[1:-1, 2:], mp[:-2, 1:-1], mp[2:, 1:-1]
    opposite = (xs ^ ys) < 0
    d1 = np.where(opposite, mp[:-2, 2:], mp[:-2, :-2])
    d2 = np.where(opposite, mp[2:, :-2], mp[2:, 2:])
    horiz = y < tg22x
    vert = (~horiz) & (y > tg67x)
    diag = (~horiz) & (~vert)
    keep = (horiz & (m > left) & (m >= right)) | (vert & (m > up) & (m >= down)) | (diag & (m > d1) & (m > d2))
    keep &= m > low
    strong = keep & (m > high)
    return strong, keep & ~strong


def canny(img: np.ndarray, low_threshold: float = 100, high_threshold: float = 200) -> np.ndarray:
    strong, weak = canny_classes(img, low_threshold, high_threshold)
    edge = strong.copy()
    while True:                                         # hysteresis: 8-connected growth into the weak pixels
        e = np.pad(edge, 1)
        nb = e[:-2, :-2] | e[:-2, 1:-1] | e[:-2, 2:] | e[1:-1, :-2] | e[1:-1, 2:] | e[2:, :-2] | e[2:, 1:-1] | e[2:, 2:]
        new = edge | (weak & nb)
        if (new == edge).all():
            return (edge * 255).astype(np.uint8)
        edge = new


def left_pad_captions(caption_embs, emb_masks):
    """sample_t2i.py:146-156 restated with torch ops: the valid tokens (a prefix, T5 pads on the right) are rotated to the END of the
    sequence, the mask is flipped."""
    import torch
    new_masks = torch.flip(emb_masks, dims=[-1])
    out = []
    for emb, mask in zip(caption_embs, emb_masks):
        v = int(mask.sum().item())
        out.append(torch.cat([emb[v:], emb[:v]]))
    return torch.stack(out), new_masks
