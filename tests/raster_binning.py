"""Exact host restatement of the rasterizer's tile binning (test helper): K1's per-Gaussian tile rects and per-tile counts, K2's
scan (tile ranges, capacity cut, status words), and the per-tile list order K3 + K4 produce.

Everything is integer (numpy int64 / uint64) except the rect, which is recomputed in float32 with the operations of
preprocess_one (csrc/raster.cu): trunc((pixx - r) / 16) and trunc(((pixx + r) + 15) / 16), each operation rounded to nearest as
numpy's float32 arithmetic is, clamped to [0, gx] / [0, gy].  The inputs are what a forward leaves behind in its own buffers
(each Gaussian's xy, radius and depth bits), so no tolerance is involved anywhere: a result either matches or it does not.

The list order is upstream's: instances ordered by (frame * T + tile, depth bits, Gaussian index), i.e. one stable sort of the
64-bit key (global tile << 32 | depth bits) over the instances generated in index order.
"""
import numpy as np

TILE = 16
SEG = 256                 # list positions per backward segment (status[2] counts them)
LONG = 2048               # lists of at least this many entries go to the long sort instance (status[13] counts them)
CTA = 256                 # Gaussians per K1 / K3 CTA, which count into one shared-memory tile table
I32_MAX = 0x7FFFFFFF


def grid(H, W):
    gx, gy = -(-W // TILE), -(-H // TILE)
    return gx, gy, gx * gy


def rects(xy, radii, H, W):
    """[N, 4] int64 (xmin, ymin, xmax, ymax) tile rects of Gaussians at pixel centres xy [N, 2] (float32) with radii [N]."""
    gx, gy, _ = grid(H, W)
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    r = np.asarray(radii).reshape(-1).astype(np.float32)
    s, f = np.float32(TILE), np.float32(15.0)
    out = np.empty((xy.shape[0], 4), np.int64)
    for a, hi in ((0, gx), (1, gy)):
        p = xy[:, a]
        lo_v = np.trunc((p - r) / s)
        hi_v = np.trunc(((p + r) + f) / s)
        out[:, a] = np.clip(lo_v.astype(np.int64), 0, hi)
        out[:, 2 + a] = np.clip(hi_v.astype(np.int64), 0, hi)
    return out


def scan(count, T, capacity):
    """K2 over the per-(frame, tile) counts [B * T]: global ranges [B * T, 2] and the status words it writes, as a dict
    {word index: value}.  A tile whose end lies past `capacity`, or that is empty, gets (0, 0)."""
    c = np.asarray(count, np.int64).reshape(-1)
    n = c.size
    B = n // T
    end = np.cumsum(c)
    start = end - c
    fits = end <= int(capacity)
    live = fits & (c > 0)
    ranges = np.zeros((n, 2), np.int64)
    ranges[live, 0], ranges[live, 1] = start[live], end[live]
    total = int(end[-1]) if n else 0
    words = {0: min(total, I32_MAX), 1: int(total > int(capacity)), 2: int(((c[live] + SEG - 1) // SEG).sum()), 3: int(live.sum()),
             13: int((live & (c >= LONG)).sum())}
    for b in range(B):
        words[4 + b] = min(int(start[b * T]), I32_MAX)
    words[4 + B] = words[0]
    return ranges, words


def restate(B, P, H, W, capacity, xy, radii, depth):
    """The binning of B frames of P Gaussians each (P includes a scene's static set), from each Gaussian's xy [B, P, 2] (float32),
    radius [B, P] and depth [B, P] (float32; only the bits are used).  Returns a dict of numpy arrays:
      rect [B, P, 4], tiles_touched [B, P], tile_count [B, T], ranges [B * T, 2] (global), words {status index: value},
      point_list [total] (per-frame Gaussian index in list order; frames follow each other), keys [total] (global tile << 32 |
      depth bits, in list order), cta_tiles [B, ceil(P / 256)] (distinct tiles each K1 / K3 CTA's rects touch) and
      instances (the total)."""
    gx, gy, T = grid(H, W)
    xy = np.asarray(xy, np.float32).reshape(B * P, 2)
    radii = np.asarray(radii).reshape(B * P)
    dbits = np.ascontiguousarray(np.asarray(depth, np.float32).reshape(B * P)).view(np.uint32).astype(np.uint64)
    rc = rects(xy, radii, H, W)
    w = rc[:, 2] - rc[:, 0]
    area = w * (rc[:, 3] - rc[:, 1])
    # instances in (frame, index) order, each Gaussian's tiles row by row
    gid = np.repeat(np.arange(B * P, dtype=np.int64), area)
    first = np.cumsum(area) - area
    k = np.arange(gid.size, dtype=np.int64) - first[gid]
    wg = w[gid]
    tile = (rc[gid, 1] + k // np.maximum(wg, 1)) * gx + rc[gid, 0] + k % np.maximum(wg, 1)
    frame = gid // P
    gtile = frame * T + tile
    count = np.bincount(gtile, minlength=B * T).astype(np.int64)
    ranges, words = scan(count, T, capacity)
    key = (gtile.astype(np.uint64) << np.uint64(32)) | dbits[gid]
    order = np.argsort(key, kind="stable")
    il = gid % P
    ncta = -(-P // CTA) if P else 0
    cta = frame * ncta + il // CTA
    pairs = np.unique(cta * np.int64(T) + tile) if gid.size else np.zeros(0, np.int64)
    cta_tiles = np.bincount(pairs // T, minlength=B * ncta).reshape(B, ncta)
    return dict(rect=rc.reshape(B, P, 4), tiles_touched=area.reshape(B, P), tile_count=count.reshape(B, T), ranges=ranges, words=words,
                point_list=il[order], keys=key[order], cta_tiles=cta_tiles, instances=int(gid.size), gx=gx, gy=gy, T=T)
