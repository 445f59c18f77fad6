"""CPU restatement of the marching cubes of neuralbody_b200/csrc/nb_mcubes.cu (vectorised numpy; TEST INFRASTRUCTURE ONLY).

Same table (tools/gen_mc_table.py), same output order, same fp64 arithmetic, so the GPU result must equal this one bit
for bit:
  * point p = (i, j, k) of an (nx, ny, nz) C-order grid owns the edges p -> p + e_a (a = x, y, z); an edge is crossed
    when exactly one end is inside (value > isovalue, compared in fp64).  A grid without cells (a dimension of 1) has
    no surface;
  * vertices follow grid-point order, x / y / z within a point; the vertex of edge p -> q along a is
    p + t e_a with t = (iso - v(p)) / (v(q) - v(p)) in fp64;
  * triangles follow the order of the cells' min corners, table order within a cell."""
import numpy as np

from tools import gen_mc_table

_TABLE = gen_mc_table.build_table()
NUM_TRIS = np.array([len(t) for t in _TABLE], np.int64)
TRIS = np.full((256, 3 * gen_mc_table.MAX_TRIS), -1, np.int64)
for _c, _t in enumerate(_TABLE):
    _flat = [e for tri in _t for e in tri]
    TRIS[_c, :len(_flat)] = _flat
EDGE_AXIS = np.array([gen_mc_table.edge_axis(e) for e in range(12)], np.int64)
EDGE_OFFSET = np.array([gen_mc_table.edge_offset(e) for e in range(12)], np.int64)
CORNERS = np.array([gen_mc_table.corner_offset(v) for v in range(8)], np.int64)


def _popcount3(m):
    return (m & 1) + ((m >> 1) & 1) + ((m >> 2) & 1)


def marching_cubes(volume, isovalue):
    """volume (nx, ny, nz) float32 -> (vertices (V,3) float64 in index coordinates, triangles (F,3) int64)."""
    v32 = np.ascontiguousarray(volume, dtype=np.float32)
    vol = v32.astype(np.float64)
    iso = float(isovalue)
    nx, ny, nz = vol.shape
    if min(nx, ny, nz) < 2:
        return np.zeros((0, 3), np.float64), np.zeros((0, 3), np.int64)
    inside = vol > iso
    mask = np.zeros(vol.shape, np.int64)
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        crossed = inside[tuple(lo)] != inside[tuple(hi)]
        mask[tuple(lo)] |= crossed.astype(np.int64) << a
    flat_mask = mask.reshape(-1)
    nv = _popcount3(flat_mask)
    vert_off = np.concatenate([[0], np.cumsum(nv)[:-1]]) if nv.size else nv

    # vertices: (point, axis) pairs in point-major, axis-minor order
    pts_idx, axes = [], []
    for a in range(3):
        p = np.nonzero((flat_mask >> a) & 1)[0]
        pts_idx.append(p)
        axes.append(np.full(p.shape, a, np.int64))
    pts_idx, axes = np.concatenate(pts_idx), np.concatenate(axes)
    order = np.argsort(pts_idx * 3 + axes, kind="stable")
    pts_idx, axes = pts_idx[order], axes[order]
    ijk = np.stack(np.unravel_index(pts_idx, vol.shape), 1)
    q = ijk.copy()
    q[np.arange(len(q)), axes] += 1
    fp = vol.reshape(-1)[pts_idx]
    fq = vol[q[:, 0], q[:, 1], q[:, 2]]
    t = (iso - fp) / (fq - fp)
    verts = ijk.astype(np.float64)
    verts[np.arange(len(verts)), axes] += t

    # triangles: cells (min corner p) in point order, table order within a cell
    cin = inside.astype(np.int64)
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for v, (dx, dy, dz) in enumerate(CORNERS):
        case |= cin[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] << v
    ntri = NUM_TRIS[case]
    cells = np.stack(np.nonzero(ntri), 1)                     # C order == point order of the min corners
    ccase = case[cells[:, 0], cells[:, 1], cells[:, 2]]
    edges = TRIS[ccase]                                        # (ncells, 15), -1 padded
    valid = edges >= 0
    e = np.where(valid, edges, 0)
    owner = cells[:, None, :] + EDGE_OFFSET[e]                 # (ncells, 15, 3)
    oflat = np.ravel_multi_index((owner[..., 0], owner[..., 1], owner[..., 2]), vol.shape)
    ax = EDGE_AXIS[e]
    omask = flat_mask[oflat]
    rank = np.where(ax > 0, omask & 1, 0) + np.where(ax > 1, (omask >> 1) & 1, 0)
    vid = vert_off[oflat] + rank
    tris = vid[valid].reshape(-1, 3)
    return verts, tris.astype(np.int64)


def counts(volume, isovalue):
    """(n_vertices, n_triangles) without building the mesh."""
    vol = np.ascontiguousarray(volume, dtype=np.float32).astype(np.float64)
    nx, ny, nz = vol.shape
    if min(nx, ny, nz) < 2:
        return 0, 0
    inside = vol > float(isovalue)
    nv = 0
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        nv += int((inside[tuple(lo)] != inside[tuple(hi)]).sum())
    cin = inside.astype(np.int64)
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for v, (dx, dy, dz) in enumerate(CORNERS):
        case |= cin[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] << v
    return nv, int(NUM_TRIS[case].sum())


# ----------------------------------------------------------------------------- mesh checks
def closed_manifold_report(tris):
    """Every undirected edge is used by exactly two triangles, once in each direction -> (ok, message)."""
    tris = np.asarray(tris, np.int64)
    if len(tris) == 0:
        return True, "empty"
    d = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]], 0)
    n = int(tris.max()) + 1
    key = d[:, 0] * n + d[:, 1]
    uniq, cnt = np.unique(key, return_counts=True)
    if (cnt != 1).any():
        return False, "%d directed edges used more than once" % int((cnt != 1).sum())
    rev = d[:, 1] * n + d[:, 0]
    missing = ~np.isin(rev, uniq)
    if missing.any():
        return False, "%d directed edges without their opposite" % int(missing.sum())
    return True, "closed"


def signed_volume(verts, tris):
    """Volume enclosed by a closed mesh (positive when the normals point outwards)."""
    a, b, c = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def pad_cube(inside, sigma, pad=10):
    """The mesh renderer's cube (if_mesh_renderer.py:42-47): float64 zeros, sigma scattered into the inside points,
    padded by `pad` zeros on every side."""
    cube = np.zeros(inside.shape)
    cube[inside == 1] = sigma
    return np.pad(cube, pad, mode="constant")
