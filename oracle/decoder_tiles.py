"""Point sets whose tensor-core decoder tiles are known in advance, for tests/test_decoder_rows_*.py.  Test infrastructure only.

The frame: out_sh (d, h, w) = (97, 97, 385), so that the four levels are 49 x 49 x 193, 25 x 25 x 97, 13 x 13 x 49 and
7 x 7 x 25 voxels and a level-l grid coordinate is exactly the level-0 one divided by 2^l.  Points are placed at level-0
cell centres (n + 0.5 per axis): on every level their coordinates then sit at least 1/16 of a voxel away from a cell
boundary, so no rounding of the world -> grid transform can move a point to another cell.

Occupancy (the voxels of a level that are non-zero) is laid out along x (level-0 units) so that a point's class, its finest
occupied level, is set by where it lies:
    level 3 everywhere; level 2 from voxel x 19 (points x >= 72); level 1 from voxel x 60 (points x >= 118), and also
    voxels x <= 10, z >= 18 (points x < 22, z >= 34: levels 3 and 1 occupied, 2 not); level 0 from voxel x 150 (x >= 149)
=> class 3 for x < 72, class 2 for 72 <= x < 118, class 1 for 118 <= x < 149, class 0 beyond, class 1 with a level gap in
the corner band.  A point with x < -9 has no occupied cell on any level (skipped, or listed as class 3 without skipping).

classify_points_kernel appends each 256-point block's entries of one class contiguously in point order, and each class's
list is a run of such block chunks.  So if the points are made of GROUPS of 128 points of one class each, every block
contributes a multiple of 128 entries to each class, every tile is one group whatever order the blocks land in, and every
half tile is 64 consecutive points of a group.  `tile_stats` predicts the decoder's counters from that.
"""
import math

import numpy as np
import torch

OUT_SH = (97, 97, 385)                          # d, h, w
LEVEL_CHANNELS = (32, 64, 128, 128)
N0 = (193, 49, 49)                              # level-0 voxels along x, y, z
VOXEL = (0.005, 0.005, 0.005)
NV = (64, 64, 128, 128)                         # staged voxels per half tile on li = 3 - level (NV_COARSE, NV_FINE)
KSTEPS = (22, 20, 16, 8)                        # layer-0 K-steps of a class-c tile (nb_layout.h class_ksteps)
TP = 128


def level_size(l):
    """(x, y, z) voxels of level l."""
    return tuple((n - 1) // (1 << l) + 1 for n in N0)


def nonzero_mask(l):
    """(z, y, x) bool: the voxels of level l that hold non-zero features."""
    X, Y, Z = level_size(l)
    z, y, x = torch.meshgrid(torch.arange(Z), torch.arange(Y), torch.arange(X), indexing="ij")
    if l == 3:
        return torch.ones((Z, Y, X), dtype=torch.bool)
    if l == 2:
        return x >= 19
    if l == 1:
        return (x >= 60) | ((x <= 10) & (z >= 18))
    return x >= 150


def make_volumes(seed, batch=1):
    """Four (B,C,D,H,W) float32 volumes: fp16-representable U(0.05, 1) on the non-zero voxels, exact zeros elsewhere."""
    g = torch.Generator().manual_seed(seed)
    vols = []
    for l, C in enumerate(LEVEL_CHANNELS):
        m = nonzero_mask(l)
        v = (torch.rand((batch, C) + tuple(m.shape), generator=g) * 0.95 + 0.05) * m
        vols.append(v.to(torch.float16).float().contiguous())
    return vols


def frame(seed=0):
    """A non-identity pose: R, Th, bounds (min corner; the max corner is min + voxel * out_sh) of one frame."""
    rng = np.random.default_rng(seed)
    rv = np.array([0.3, -0.2, 0.1]) + rng.uniform(-0.2, 0.2, 3)
    th = np.array([0.1, 0.2, 1.0]) + rng.uniform(-0.3, 0.3, 3)
    a = np.linalg.norm(rv)
    k = rv / a
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + math.sin(a) * Kx + (1 - math.cos(a)) * Kx @ Kx
    lo = np.array([-0.45, -0.12, -0.2]) + rng.uniform(-0.05, 0.05, 3)
    ext = np.array([VOXEL[0] * OUT_SH[2], VOXEL[1] * OUT_SH[1], VOXEL[2] * OUT_SH[0]])
    bounds = np.stack([lo, lo + ext])
    return (torch.tensor(R, dtype=torch.float32), torch.tensor(th, dtype=torch.float32)[None],
            torch.tensor(bounds, dtype=torch.float32))


def world_points(q0, R, Th, bounds):
    """Level-0 grid coordinates (P,3) (x, y, z) -> world points (P,3) float32 of the frame (c = (w - Th) R)."""
    return T_world(q0, R, Th, bounds).float()


# ------------------------------------------------------------------------------------------------ structure of a point
def _cells(q0, l):
    return torch.floor(torch.as_tensor(q0, dtype=torch.float64) / (1 << l)).long()


def occupied(q0, l):
    """(P,) bool: the level-l cell of each point holds a non-zero voxel (the decoder's cell bitmap)."""
    f = _cells(q0, l)
    size = level_size(l)
    m = nonzero_mask(l)
    ok = torch.ones(f.shape[0], dtype=torch.bool)
    for a in range(3):
        ok &= (f[:, a] >= -1) & (f[:, a] <= size[a])
    occ = torch.zeros(f.shape[0], dtype=torch.bool)
    for c in range(8):
        v = f + torch.tensor([c & 1, (c >> 1) & 1, c >> 2])
        inr = ok.clone()
        for a in range(3):
            inr &= (v[:, a] >= 0) & (v[:, a] < size[a])
        vv = v.clone()
        for a in range(3):
            vv[:, a] = vv[:, a].clamp(0, size[a] - 1)
        occ |= inr & m[vv[:, 2], vv[:, 1], vv[:, 0]]
    return occ


def classes(q0, skip=True):
    """(P,) the list class of each point: finest occupied level, -1 = not listed (skip) / 3 (no skipping)."""
    occ = torch.stack([occupied(q0, l) for l in range(4)], 1)
    cls = torch.full((occ.shape[0],), -1, dtype=torch.long)
    for l in (3, 2, 1, 0):
        cls = torch.where(occ[:, l], torch.full_like(cls, l), cls)
    if not skip:
        cls = torch.where(cls < 0, torch.full_like(cls, 3), cls)
    return cls


def corner_ids(q0, l):
    """(P,8) voxel ids of the clamped cell's 8 corners on level l (clamped_cell in nb_render_tc_list.cu)."""
    f = _cells(q0, l)
    size = level_size(l)
    lo = []
    for a in range(3):
        i0, n = f[:, a], size[a]
        lo.append(torch.where(i0 < 0, torch.zeros_like(i0), torch.where(i0 >= n - 1, torch.full_like(i0, n - 2), i0)))
    X, Y = size[0], size[1]
    ids = [((lo[2] + (c >> 2)) * Y + lo[1] + ((c >> 1) & 1)) * X + lo[0] + (c & 1) for c in range(8)]
    return torch.stack(ids, 1)


def distinct_voxels(q0, l):
    """Distinct corner voxels of level l over the points of q0 that are occupied there (one half tile's hash)."""
    occ = occupied(q0, l)
    if not bool(occ.any()):
        return 0
    return int(torch.unique(corner_ids(q0, l)[occ]).numel())


def tile_stats(groups, skip=True):
    """The decoder's counters for a point set made of `groups` (each (<=128, 3) level-0 coordinates of one class, or of
    unlisted points): {0: tiles, 1: listed points, 4: layer-0 K-steps, 5 / 6: coarse half tiles staged / direct, 7: fine
    half tiles direct}."""
    st = {0: 0, 1: 0, 4: 0, 5: 0, 6: 0, 7: 0}
    for q in groups:
        cls = classes(q, skip)
        if bool((cls < 0).all()):
            continue
        assert bool((cls == cls[0]).all()) and q.shape[0] <= TP, "a group holds points of one class"
        c = int(cls[0])
        st[0] += 1
        st[1] += q.shape[0]
        st[4] += KSTEPS[c]
        for half in range(2):
            h = q[64 * half:64 * half + 64]
            if h.shape[0] == 0:
                continue
            for li in range(4 - c):
                n = distinct_voxels(h, 3 - li)
                if li < 2:
                    st[5 if n <= NV[li] else 6] += 1
                elif n > NV[li]:
                    st[7] += 1
    return st


def stats_by_class(cls):
    """Counters [0], [1], [4] from the per-point classes alone (any block order, any tile composition)."""
    st = {0: 0, 1: 0, 4: 0}
    for c in range(4):
        n = int((cls == c).sum())
        t = (n + TP - 1) // TP
        st[0] += t
        st[1] += n
        st[4] += t * KSTEPS[c]
    return st


# ------------------------------------------------------------------------------------------------ designed half tiles
def block_half(level, blocks, n=64):
    """n points (level-0 coordinates) whose level-`level` cells cover the disjoint voxel blocks ((x, y, z) start, (a, b, c)
    size) exactly: the half tile's distinct voxels on that level are the blocks' voxels."""
    cells = []
    for (sx, sy, sz), (a, b, c) in blocks:
        for z in range(sz, sz + c - 1):
            for y in range(sy, sy + b - 1):
                for x in range(sx, sx + a - 1):
                    cells.append((x, y, z))
    assert len(cells) <= n
    s = 1 << level
    pts = []
    for k in range(n):
        cx, cy, cz = cells[k % len(cells)]
        off = [(k * 5 + 3 * ax) % s for ax in range(3)]
        pts.append((cx * s + off[0] + 0.5, cy * s + off[1] + 0.5, cz * s + off[2] + 0.5))
    return torch.tensor(pts, dtype=torch.float64)


def blocks_exactly(level, x0, count):
    """Disjoint voxel blocks at voxel x >= x0 with exactly `count` voxels: 64 / 128 as one box, 65 / 129 as boxes that
    leave no voxel of a 2 x 2 x 2 corner block shared (27 + 18 + 12 + 8, plus a 4 x 4 x 4 box for 129)."""
    if count == 64:
        return [((x0, 0, 0), (4, 4, 4))]
    if count == 128:
        return [((x0, 0, 0), (4, 4, 8))]
    tail = [((0, 0, 0), (3, 3, 3)), ((3, 0, 0), (3, 3, 2)), ((6, 0, 0), (3, 2, 2)), ((0, 3, 0), (2, 2, 2))]
    if count == 65:
        return [((x0 + s[0], s[1], s[2]), sz) for s, sz in tail]
    assert count == 129
    return [((x0, 0, 0), (4, 4, 4))] + [((x0 + 4 + s[0], s[1] + (2 if s[1] else 0), s[2]), sz) for s, sz in tail]


# the first voxel x of each level's designs: inside the region where that level is the finest occupied one
DESIGN_X0 = {3: 0, 2: 19, 1: 59, 0: 150}


def limit_group(level, first, second):
    """One 128-point group of class `level`: half tiles with exactly `first` and `second` distinct voxels on that level."""
    x0 = DESIGN_X0[level]
    return torch.cat([block_half(level, blocks_exactly(level, x0, first)),
                      block_half(level, blocks_exactly(level, x0, second))])


REGIONS = {                 # class -> level-0 cell ranges (x, y, z) of random points of that class
    3: ((0, 70), (0, 48), (0, 30)),
    2: ((73, 117), (0, 48), (0, 48)),
    1: ((119, 148), (0, 48), (0, 48)),
    "gap": ((0, 21), (0, 48), (35, 48)),
    0: ((151, 192), (0, 48), (0, 48)),
    "empty": ((-40, -13), (0, 48), (0, 48)),
}


def random_points(region, n, seed, ymax=None):
    """n random level-0 cell centres of a region (y below ymax if given)."""
    g = torch.Generator().manual_seed(seed)
    box = list(REGIONS[region])
    if ymax is not None:
        box[1] = (box[1][0], min(box[1][1], ymax))
    cols = [torch.randint(lo, hi, (n,), generator=g) for lo, hi in box]
    return torch.stack(cols, 1).double() + 0.5


def local_points(region, n, seed, span=3):
    """n points in one span^3 box of level-0 cells of the region: a half tile of them stays staged on every level."""
    g = torch.Generator().manual_seed(seed)
    base = [int(torch.randint(lo, hi - span, (1,), generator=g)) for lo, hi in REGIONS[region]]
    cols = [b + torch.randint(0, span, (n,), generator=g) for b in base]
    return torch.stack(cols, 1).double() + 0.5


def boundary_points():
    """Points on each level's faces, edges and corners: every combination of (low face, interior, high face) per axis but
    the all-interior one, on the low-x side (class 3, or 1 in the gap band) and the high-x side (class 0)."""
    pts = []
    for xs in (-0.5, 192.5):
        for ys in (-0.5, 20.5, 48.5):
            for zs in (-0.5, 20.5, 48.5):
                if ys == 20.5 and zs == 20.5:
                    pts.append((xs, ys, zs))            # a face of x alone
                    continue
                pts.append((xs, ys, zs))
                pts.append((xs + (1.0 if xs < 0 else -1.0), ys, zs))   # next to the x face: the y / z faces and edges alone
    return torch.tensor(pts, dtype=torch.float64)


def groups_by_class(q0, skip=True):
    """Groups of exactly 128 points per class from q0, repeating points to fill the last group of a class."""
    cls = classes(q0, skip)
    out = []
    for c in (3, 2, 1, 0):
        q = q0[cls == c]
        if q.shape[0] == 0:
            continue
        reps = (q.shape[0] + TP - 1) // TP * TP
        q = q[torch.arange(reps) % q.shape[0]]
        out += list(q.split(TP))
    return out


def probe_points():
    """16 class-0 probes in one 4 x 2 x 2 box of level-0 cells, whose sigma must not depend on the tile they are decoded in.
    Beside local_points neighbours they are staged on every level; beside random_points ones, gathered directly."""
    x, y, z = torch.meshgrid(torch.arange(4), torch.arange(2), torch.arange(2), indexing="ij")
    return torch.stack([x.reshape(-1) + 170, y.reshape(-1) + 20, z.reshape(-1) + 20], 1).double() + 0.5


def half_paths(q):
    """Per level 3..0 of a half tile of points (<= 64, one class): 'staged' or 'direct' (None: the level is not gathered)."""
    c = int(classes(q)[0])
    out = []
    for li in range(4):
        if li > 3 - c:
            out.append(None)
        else:
            out.append("staged" if distinct_voxels(q, 3 - li) <= NV[li] else "direct")
    return out


# level-0 units of one level-3 voxel: translating a point set by it along y keeps its classes and distinct voxel counts
Y_STEP = 8


def render_rays(groups, R, Th, bounds, z0=1.0):
    """Rays whose 2 samples reproduce `groups` (each 128 points, y + Y_STEP < 49): in the render list a block of 512 rays
    lists sample 0 of its rays, then sample 1, so ray 128 g + i of block k carries point i of groups[4 k + g] at depth z0
    and the same point moved by Y_STEP along y at depth z0 + step.  All rays share one direction.  Returns ray_o (n,3),
    ray_d (n,3), z (n,2) float32 and the sample points' level-0 coordinates (n,2,3)."""
    q = torch.cat(groups)
    n = q.shape[0]
    shift = torch.tensor([0.0, Y_STEP, 0.0], dtype=torch.float64)
    w0 = T_world(q, R, Th, bounds)
    w1 = T_world(q + shift, R, Th, bounds)
    step = float(torch.norm(w1[0] - w0[0]))
    d = (w1[0] - w0[0]) / step
    o = w0 - d[None] * z0
    z = torch.tensor([z0, z0 + step], dtype=torch.float64).expand(n, 2)
    return o.float(), d[None].expand(n, 3).float().contiguous(), z.float().contiguous(), torch.stack([q, q + shift], 1)


def render_groups(groups):
    """The tiles of render_rays(groups): per block of 4 groups, the groups, then the same groups moved by Y_STEP."""
    shift = torch.tensor([0.0, Y_STEP, 0.0], dtype=torch.float64)
    out = []
    for k in range(0, len(groups), 4):
        blk = groups[k:k + 4]
        out += blk + [g + shift for g in blk]
    return out


def T_world(q0, R, Th, bounds):
    """world_points in float64."""
    q0 = torch.as_tensor(q0, dtype=torch.float64)
    ext = torch.tensor([VOXEL[0] * OUT_SH[2], VOXEL[1] * OUT_SH[1], VOXEL[2] * OUT_SH[0]], dtype=torch.float64)
    c = bounds[0].double() + q0 / torch.tensor([n - 1 for n in N0], dtype=torch.float64) * ext
    return c @ R.double().t() + Th.double().reshape(1, 3)
