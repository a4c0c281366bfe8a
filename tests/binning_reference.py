"""numpy restatement of the binning stage (csrc/binning.cu, csrc/radix.cuh), from the forward's own per-record outputs.

Inputs: radii [V*P], the records' pixel centres px, py and depths (GeomRec fields 0, 1 and 11), record index vp = v*P + i.
  * rect          the tile rectangle in the preprocess kernel's float32 operation order (preprocess.cu), records with radius > 0
  * tiles_touched w * h of the rect, 0 for culled records
  * depth_order   stable argsort of the u32 depth keys (the depth bits; 0 for culled records) over all V*P records, views mixed
  * offsets       inclusive sum of tiles_touched in depth order (the state keeps the low 32 bits)
  * per view      the view's records in depth order emit their rect's tiles row-major with key v*ntiles + ty*gx + tx; a stable
                  sort by that key gives sorted_tile_keys and point_list, and ranges [ntiles, 2] (zero for empty tiles)
Views occupy consecutive key ranges, so view v's part of the batch's sorted arrays is [view_start[v], view_start[v + 1]): the
per-view functions need host memory for one view only."""
import numpy as np

GS_TILE = 16
_f32 = np.float32


def _tile_index(f, g):
    # (int)f then clamp to [0, g]: clip first in float (CUDA's cast saturates, numpy's cast of an out-of-range float does not);
    # for f in (-1, 0) both give 0, and the cast truncates toward zero either way
    return np.clip(f, 0, g).astype(np.int64)


def rects(px, py, radii, gx, gy):
    """[N, 4] int64 (x0, y0, x1, y1) in the kernel's float32 order; all zero where radius <= 0."""
    px, py = np.asarray(px, _f32), np.asarray(py, _f32)
    radii = np.asarray(radii).reshape(-1)
    r = radii.astype(_f32)
    t, one = _f32(GS_TILE), _f32(1)
    out = np.stack([_tile_index((px - r) / t, gx), _tile_index((py - r) / t, gy),
                    _tile_index((((px + r) + t) - one) / t, gx), _tile_index((((py + r) + t) - one) / t, gy)], 1)
    out[radii <= 0] = 0
    return out


class BinningReference:
    """The batch-level part (rect, tiles_touched, depth keys / order, offsets, D) on construction; view(v) for the rest."""

    def __init__(self, radii, px, py, depth, H, W, V=1):
        self.radii = np.asarray(radii).reshape(-1)
        self.V = int(V)
        self.P = self.radii.size // self.V
        self.gx, self.gy = (W + GS_TILE - 1) // GS_TILE, (H + GS_TILE - 1) // GS_TILE
        self.ntiles = self.gx * self.gy
        vis = self.radii > 0
        self.rect = rects(px, py, self.radii, self.gx, self.gy)
        self.tiles_touched = np.where(vis, (self.rect[:, 2] - self.rect[:, 0]) * (self.rect[:, 3] - self.rect[:, 1]), 0).astype(np.uint32)
        bits = np.ascontiguousarray(depth, _f32).reshape(-1).view(np.uint32)
        assert not bits[~vis].any(), "culled records must carry depth 0"
        self.depth_keys = np.where(vis, bits, 0).astype(np.uint32)
        self.depth_order = np.argsort(self.depth_keys, kind="stable").astype(np.uint32)
        csum = np.cumsum(self.tiles_touched[self.depth_order], dtype=np.uint64)
        self.offsets = csum.astype(np.uint32)  # low 32 bits
        self.num_rendered = int(csum[-1]) if csum.size else 0
        per_view = self.tiles_touched.reshape(self.V, self.P).sum(1, dtype=np.int64)
        self.view_start = np.concatenate([[0], np.cumsum(per_view)]).astype(np.int64)
        # every view's records in global depth order, view after view (a stable regroup of depth_order)
        self._by_view = self.depth_order[np.argsort(self.depth_order // np.uint32(max(self.P, 1)), kind="stable")]

    def view(self, v):
        """View v: sorted_tile_keys, point_list (u32, the batch's slice) and ranges [ntiles, 2] (u32, batch positions)."""
        recs = self._by_view[v * self.P:(v + 1) * self.P].astype(np.int64)
        cnt = self.tiles_touched[recs].astype(np.int64)
        keep = cnt > 0
        recs, cnt = recs[keep], cnt[keep]
        D = int(cnt.sum())
        owner = np.repeat(np.arange(recs.size), cnt)
        local = np.arange(D, dtype=np.int64) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        x0, y0, x1, _ = (self.rect[recs, k][owner] for k in range(4))
        w = x1 - x0
        dy = local // w
        tile = (y0 + dy) * self.gx + x0 + (local - dy * w)
        s = np.argsort(tile, kind="stable")
        tile, vals = tile[s], recs[owner][s]
        counts = np.bincount(tile, minlength=self.ntiles).astype(np.int64)
        end = np.cumsum(counts) + self.view_start[v]
        ranges = np.where((counts > 0)[:, None], np.stack([end - counts, end], 1), 0)
        return dict(sorted_tile_keys=(tile + v * self.ntiles).astype(np.uint32), point_list=vals.astype(np.uint32),
                    ranges=ranges.astype(np.uint32))

    def full(self):
        """All views concatenated: the whole batch's sorted_tile_keys, point_list and ranges [V*ntiles, 2]."""
        parts = [self.view(v) for v in range(self.V)]
        return {k: np.concatenate([p[k] for p in parts]) for k in ("sorted_tile_keys", "point_list", "ranges")}


def bits_for(n):
    """Key bits of the tile sort for n = V * ntiles keys (binning.cu's bits_for)."""
    b = 0
    while (1 << b) < n:
        b += 1
    return b
