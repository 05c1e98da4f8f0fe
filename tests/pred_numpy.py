"""A plain numpy restatement of one prediction-cost job (x265cu_pred_cost_batch; the oracle's orc_pred_cost): the luma 8-tap
quarter-pel and chroma 4-tap eighth-pel interpolation of ipfilter.cpp on the pixel path (copy / hpp / vpp / hps + vsp) and the
14-bit path (p2s / hps / vps / hps + vss), in the reference's integer order; addAvg and pixelavg_pp; SAD; SATD with the
reference's tiling (satd_8x4 = (|H(left)| + |H(right)|) >> 1 over its two 4x4 halves when the width is a multiple of 8,
satd_4x4 = |H| >> 1 otherwise; every coefficient of H has the parity of the block's sum, so |H| is even and halving each half
first would give the same value).  It is slow on purpose: it serves as a third opinion on hundreds of jobs and to state what a
job reads (read rectangles per plane) and which clips it engages.

Planes are 2-D arrays (rows x stride) with the picture's pixel (0, 0) at (oy, ox); vectors are quarter-pel, used as eighth-pel
for the half-resolution chroma planes (4:2:0)."""
import numpy as np

LUMA_TAPS = np.array([[0, 0, 0, 64, 0, 0, 0, 0], [-1, 4, -10, 58, 17, -5, 1, 0],
                      [-1, 4, -11, 40, 40, -11, 4, -1], [0, 1, -5, 17, 58, -10, 4, -1]], np.int64)
CHROMA_TAPS = np.array([[0, 64, 0, 0], [-2, 58, 10, -2], [-4, 54, 16, -2], [-6, 46, 28, -4],
                        [-4, 36, 36, -4], [-4, 28, 46, -6], [-2, 16, 54, -4], [-2, 10, 58, -2]], np.int64)
OFFS = 8192                                         # IF_INTERNAL_OFFS


def read_rect(x, y, w, h, mv, ntaps):
    """Picture-coordinate rectangle (x0, y0, x1, y1), inclusive, that one plane's prediction of the w x h block at (x, y) reads"""
    fb = 2 if ntaps == 8 else 3
    ix, iy = x + (mv[0] >> fb), y + (mv[1] >> fb)
    xf, yf = mv[0] & ((1 << fb) - 1), mv[1] & ((1 << fb) - 1)
    hl = ntaps // 2 - 1
    x0, x1 = (ix - hl, ix + w - 1 + ntaps // 2) if xf else (ix, ix + w - 1)
    y0, y1 = (iy - hl, iy + h - 1 + ntaps // 2) if yf else (iy, iy + h - 1)
    return x0, y0, x1, y1


def _taps_sum(win, taps, axis, n):
    """sum_k win[k : k + n] * taps[k] along `axis` (int64)"""
    out = 0
    for k, c in enumerate(taps):
        out = out + (win[k:k + n, :] if axis == 0 else win[:, k:k + n]) * int(c)
    return out


def predict(plane, oy, ox, x, y, w, h, mv, ntaps, depth, short, stats=None):
    """One plane's prediction of the w x h block at picture (x, y): pixel values (short=False) or the 14-bit intermediate.
    stats (a dict) collects whether the pixel-path clip engaged below 0 ('interp_lo') or above maxv ('interp_hi')."""
    maxv = (1 << depth) - 1
    head = 14 - depth
    x0, y0, x1, y1 = read_rect(x, y, w, h, mv, ntaps)
    assert y0 + oy >= 0 and x0 + ox >= 0 and y1 + oy < plane.shape[0] and x1 + ox < plane.shape[1], "read outside the allocation"
    win = plane[y0 + oy:y1 + oy + 1, x0 + ox:x1 + ox + 1].astype(np.int64)
    fb = 2 if ntaps == 8 else 3
    xf, yf = mv[0] & ((1 << fb) - 1), mv[1] & ((1 << fb) - 1)
    tab = LUMA_TAPS if ntaps == 8 else CHROMA_TAPS

    def clip(v):
        if stats is not None:
            stats["interp_lo"] = stats.get("interp_lo", False) or bool((v < 0).any())
            stats["interp_hi"] = stats.get("interp_hi", False) or bool((v > maxv).any())
        return np.clip(v, 0, maxv)
    if not xf and not yf:
        return (win << head) - OFFS if short else win                                   # p2s / copy_pp
    if not yf:
        s = _taps_sum(win, tab[xf], 1, w)
        return (s + (-OFFS << (6 - head))) >> (6 - head) if short else clip((s + 32) >> 6)     # hps / hpp
    if not xf:
        s = _taps_sum(win, tab[yf], 0, h)
        return (s + (-OFFS << (6 - head))) >> (6 - head) if short else clip((s + 32) >> 6)     # vps / vpp
    mid = (_taps_sum(win, tab[xf], 1, w) + (-OFFS << (6 - head))) >> (6 - head)       # hps, row-extended
    s = _taps_sum(mid, tab[yf], 0, h)
    if short:
        return s >> 6                                                                   # vss
    sh = 6 + head
    return clip((s + (1 << (sh - 1)) + (OFFS << 6)) >> sh)                              # vsp


def add_avg(a, b, depth, stats=None):
    """Yuv::addAvg of two 14-bit predictions (pixel.cpp addAvg)"""
    sh = 15 - depth
    v = (a + b + (1 << (sh - 1)) + 2 * OFFS) >> sh
    if stats is not None:
        stats["avg_lo"] = stats.get("avg_lo", False) or bool((v < 0).any())
        stats["avg_hi"] = stats.get("avg_hi", False) or bool((v > (1 << depth) - 1).any())
    return np.clip(v, 0, (1 << depth) - 1)


def pixelavg_pp(a, b):
    return (a + b + 1) >> 1


def sad(a, b):
    return int(np.abs(a.astype(np.int64) - b.astype(np.int64)).sum())


_H4 = np.array([[1, 1, 1, 1], [1, -1, 1, -1], [1, 1, -1, -1], [1, -1, -1, 1]], np.int64)


def _had4(d):
    """sum of |coefficients| of the unnormalised 4x4 Hadamard transform of d"""
    return int(np.abs(_H4 @ d @ _H4.T).sum())


def satd(a, b):
    d = a.astype(np.int64) - b.astype(np.int64)
    h, w = d.shape
    acc = 0
    for ty in range(0, h, 4):
        if w % 8 == 0:
            for tx in range(0, w, 8):
                acc += (_had4(d[ty:ty + 4, tx:tx + 4]) + _had4(d[ty:ty + 4, tx + 4:tx + 8])) >> 1    # satd_8x4
        else:
            for tx in range(0, w, 4):
                acc += _had4(d[ty:ty + 4, tx:tx + 4]) >> 1                                            # satd_4x4
    return acc


def pred_cost(pics, job, chroma_planes=True):
    """(cost, reads, stats) of one x265cu_pred_job record on `pics` (pred_helpers.Pics).  reads: [(plane name, x0, y0, x1, y1)]
    in picture coordinates of that plane; stats: the clips engaged ('interp_lo' / 'interp_hi' / 'avg_lo' / 'avg_hi')."""
    depth = pics.depth
    py, px = divmod(int(job["offset"]), pics.stride)
    w, h = int(job["pw"]), int(job["ph"])
    lists = [(int(job["ref0"]), [int(v) for v in job["mv0"]]), (int(job["ref1"]), [int(v) for v in job["mv1"]])]
    lists = [(r, mv) for r, mv in lists if r >= 0]
    bi = len(lists) == 2
    avgpp = bool(job["flags"] & 2)
    cw, ch = w >> 1, h >> 1
    chroma = bool(job["flags"] & 1) and chroma_planes and cw % 4 == 0 and ch % 4 == 0 and not (bi and avgpp)
    oy, ox = divmod(pics.org, pics.stride)
    coy, cox = divmod(pics.corg, pics.cstride)
    reads, stats = [], {}

    def plane_pred(r, mv, p, short):
        if p == 0:
            reads.append(("luma", *read_rect(px, py, w, h, mv, 8)))
            return predict(pics.refs2d[r], oy, ox, px, py, w, h, mv, 8, depth, short, stats)
        reads.append(("cb" if p == 1 else "cr", *read_rect(px >> 1, py >> 1, cw, ch, mv, 4)))
        return predict(pics.rc2d[r][p - 1], coy, cox, px >> 1, py >> 1, cw, ch, mv, 4, depth, short, stats)

    preds = []
    for p in range(3 if chroma else 1):
        if not bi:
            preds.append(plane_pred(*lists[0], p, False))
        elif avgpp:
            preds.append(pixelavg_pp(plane_pred(*lists[0], p, False), plane_pred(*lists[1], p, False)))
        else:
            preds.append(add_avg(plane_pred(*lists[0], p, True), plane_pred(*lists[1], p, True), depth, stats))
    src = pics.fenc2d[oy + py:oy + py + h, ox + px:ox + px + w]
    if job["cost"] == 0:
        return sad(src, preds[0]), reads, stats
    cost = satd(src, preds[0])
    for p in (1, 2) if chroma else ():
        cost += satd(pics.fc2d[p - 1][coy + (py >> 1):coy + (py >> 1) + ch, cox + (px >> 1):cox + (px >> 1) + cw], preds[p])
    return cost, reads, stats
