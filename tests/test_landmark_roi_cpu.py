"""The frame rectangle FaceLandmark uploads for a face in a host frame (crop_read_rects) holds every frame pixel the crop
reads.  The pixels read come from a scalar restatement of the crop: oracle crop_geometry, the end clamps of numpy slicing
on the padded frame, and the tap indices of cv2.resize (_linear_taps), both taps of every output pixel."""
import functools

import numpy as np

S = 256


@functools.lru_cache(maxsize=None)
def _taps(src, clamp_x):
    """Every source index that one of the two taps of some destination index of an S-wide resize from src reads."""
    from oracle.host_ref import _linear_taps
    idx, _, _ = _linear_taps(S, src, clamp_x)
    if clamp_x:
        both = np.concatenate([idx, np.minimum(idx + 1, src - 1)])
    else:
        both = np.concatenate([np.clip(idx, 0, src - 1), np.clip(idx + 1, 0, src - 1)])
    return np.unique(both).astype(np.int64)


def _read_range(box, H, W, extend0):
    """((x_lo, x_hi), (y_lo, y_hi)) inclusive of the frame pixels the crop reads, None when it reads none; and the
    crop's columns and rows in frame coordinates (cx0, cw, cy0, ch), None for a box too small or empty."""
    from oracle.host_ref import crop_geometry
    g = crop_geometry(box, extend0, 20)
    if g is None:
        return None, None
    add, x1, y1, x2, y2 = g
    x1, y1 = max(x1, 0), max(y1, 0)
    x2, y2 = min(x2, W + 2 * add), min(y2, H + 2 * add)
    w, h = x2 - x1, y2 - y1
    if w <= 0 or h <= 0:
        return None, None
    # crop column t is frame column x1 - add + t (outside the frame: the zero border, not read); a pixel is read when
    # both its column and its row are in the frame
    fx = x1 - add + _taps(w, True)
    fy = y1 - add + _taps(h, False)
    fx, fy = fx[(fx >= 0) & (fx < W)], fy[(fy >= 0) & (fy < H)]
    span = (x1 - add, w, y1 - add, h)
    if not len(fx) or not len(fy):
        return None, span
    return ((int(fx.min()), int(fx.max())), (int(fy.min()), int(fy.max()))), span


def _random_cases(rng, n):
    sizes = [(1, 1), (1, 7), (5, 1), (2, 3), (19, 23), (64, 48), (273, 410), (480, 640), (1080, 1920), (2160, 3840)]
    out = []
    for _ in range(n):
        H, W = sizes[rng.integers(len(sizes))]
        kind = rng.integers(4)
        if kind == 0:                                   # small: sides around the 20 px cut
            bw, bh = rng.uniform(1, 40, 2)
        elif kind == 1:                                 # larger than the frame
            bw, bh = rng.uniform(1, 3, 2) * max(H, W) + 21
        else:
            bw, bh = rng.uniform(15, 1.2 * max(H, W, 30), 2)
        x0 = rng.uniform(-1.5 * bw - 5, W + 5)           # hanging over every edge, wholly outside, inside
        y0 = rng.uniform(-1.5 * bh - 5, H + 5)
        if rng.integers(8) == 0:
            x0, bw = np.round(x0), np.round(bw)          # integral coordinates too
        out.append((H, W, np.array([x0, y0, x0 + bw, y0 + bh], np.float32)))
    return out


def test_roi_holds_every_pixel_the_crop_reads():
    from peppa_pig_face_landmark_b200.core.api.face_landmark import crop_read_rects, face_scale
    from peppa_pig_face_landmark_b200.core.api.facer import get_cfg
    kcfg = get_cfg()['Skps']['Keypoints']
    extend0, fs = kcfg['base_extend_range'][0], face_scale(kcfg)
    rng = np.random.default_rng(2024)
    cases = _random_cases(rng, 100_000)
    by_frame = {}
    for i, (H, W, b) in enumerate(cases):
        by_frame.setdefault((H, W), []).append(i)
    rects = np.zeros((len(cases), 4), np.int64)
    for (H, W), idx in by_frame.items():
        rects[idx] = crop_read_rects(np.stack([cases[i][2] for i in idx]), H, W, fs)
    seen = {"read": 0, "small": 0, "outside": 0, "edge": 0, "tiny_frame": 0, "huge": 0}
    for (H, W, b), r in zip(cases, rects):
        rng_read, span = _read_range(b, H, W, extend0)
        x0, y0, x1, y1 = (int(v) for v in r)
        if rng_read is None:
            if span is None:
                seen["small"] += 1
                assert (x0, y0, x1, y1) == (0, 0, 0, 0), (H, W, b, r)
            elif not (span[0] < W and span[0] + span[1] > 0 and span[2] < H and span[2] + span[3] > 0):
                seen["outside"] += 1
                assert (x0, y0, x1, y1) == (0, 0, 0, 0), (H, W, b, r)
            continue
        seen["read"] += 1
        seen["tiny_frame"] += H * W <= 4
        seen["huge"] += b[2] - b[0] > W and b[3] - b[1] > H
        (xl, xh), (yl, yh) = rng_read
        seen["edge"] += xl == 0 or yl == 0 or xh == W - 1 or yh == H - 1
        assert 0 <= x0 <= xl and xh < x1 <= W and 0 <= y0 <= yl and yh < y1 <= H, (H, W, b, r, rng_read)
        # and no more than the crop's rectangle widened by one pixel
        cx0, cw, cy0, ch = span
        assert x0 >= cx0 - 1 and x1 <= cx0 + cw + 1 and y0 >= cy0 - 1 and y1 <= cy0 + ch + 1, (H, W, b, r, span)
    assert min(seen.values()) > 100, seen


def test_roi_of_a_300px_face():
    """A 300-px face reads a rectangle of 1.4 * 300 px, plus one on each side."""
    from peppa_pig_face_landmark_b200.core.api.face_landmark import crop_read_rects
    r = crop_read_rects(np.array([[700, 300, 1000, 600]], np.float32), 1080, 1920, float(np.float32(1.4)))[0]
    assert (r[2] - r[0], r[3] - r[1]) == (422, 422)
