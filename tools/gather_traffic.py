"""Layer-0 gather traffic of the tensor-core decoder, counted on the CPU (no GPU needed).

Replays what the list pipeline does with one view of a synthetic scene (oracle/synth.py): the samples of every ray, their
four cell-occupancy bits and class (finest occupied level), the class lists in the classifier's order (blocks of
1024 / S rays, sample-major, one class after the other), and 128-row tiles of two 64-row halves.  For every level it
prints the corner-vector bytes the gather requests (8 per occupied row), the bytes of the distinct voxels per tile, and
the distribution of distinct voxels per half tile, and the share of half tiles that do not fit the decoder's staging of
--nv voxels (coarse levels 3 and 2) or --nv-fine voxels (fine levels 1 and 0); the decoder gathers those directly from
global memory.

    python tools/gather_traffic.py [--size 512] [--samples 64] [--nv 64] [--nv-fine 128]

The feature volumes are the scene's dense synthetic ones: a voxel is occupied when any of its channels is non-zero."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TP, HALF = 128, 64


def corner_cells(g, dims):
    """grid coords (N, 3) in [-1, 1] (x, y, z) -> (clamped low corner voxel id (N,), in-bounds cell index (N,) or -1), as the
    decoder's clamped_cell / the classifier's cell test compute them"""
    D, H, W = dims
    base = np.zeros(len(g), np.int64)
    ok = np.ones(len(g), bool)
    cell = np.zeros(len(g), np.int64)
    for axis, size, stride, cstride in ((0, W, 1, 1), (1, H, W, W + 1), (2, D, W * H, (W + 1) * (H + 1))):
        i = ((g[:, axis] + 1.0) * 0.5 * (size - 1)).astype(np.float32)
        f = np.floor(i)
        ok &= (f >= -1) & (f <= size - 1)           # (f == size: every corner is outside, the cell holds nothing)
        i0 = np.where(np.isfinite(f), f, -2).astype(np.int64)
        c = np.where(i0 < 0, 0, np.where(i0 >= size - 1, size - 2, i0))      # the clamped low corner on this axis
        base += c * stride
        cell += (i0 + 1) * cstride
    return base, np.where(ok, cell, -1)


def replay(size, n_samples):
    from oracle import synth, neuralbody_oracle as O
    scene = synth.make_scene(H=size, W=size, scale=1.0, all_hit=True)
    sp = O.prepare_sp_input(scene)
    wpts, _ = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], n_samples)
    n = wpts.shape[1]
    can = O.pts_to_can_pts(wpts.reshape(1, -1, 3), scene["R"], scene["Th"])
    g = O.get_grid_coords(can, scene["bounds"], sp["out_sh"], scene["voxel_size"])[0].numpy()
    levels = []
    lm = np.zeros(len(g), np.int64)
    for lvl, v in enumerate(scene["volumes"]):
        C, D, H, W = v.shape[1:]
        base, cell = corner_cells(g, (D, H, W))
        vox = (v[0].abs().sum(0) > 0).numpy()                                  # (D, H, W)
        pad = np.zeros((D + 2, H + 2, W + 2), bool)
        pad[1:-1, 1:-1, 1:-1] = vox
        occ = np.zeros((D + 1, H + 1, W + 1), bool)                             # cell (cz, cy, cx): OR of its 8 corners
        for dz in (0, 1):
            for dy in (0, 1):
                for dx in (0, 1):
                    occ |= pad[dz:dz + D + 1, dy:dy + H + 1, dx:dx + W + 1]
        bit = np.zeros(len(g), bool)
        ok = cell >= 0
        bit[ok] = occ.reshape(-1)[cell[ok]]
        lm |= bit.astype(np.int64) << lvl
        levels.append(dict(C=C, dims=(D, H, W), base=base))
    # list order: blocks of rpg rays, sample-major inside a block, the block's entries of a class contiguous
    rpg = 1024 // n_samples
    ids = np.arange(n * n_samples).reshape(n, n_samples)                       # sample id = ray * S + s
    nblk = (n + rpg - 1) // rpg
    order = np.full((nblk * rpg, n_samples), -1, np.int64)
    order[:n] = ids
    order = order.reshape(nblk, rpg, n_samples).transpose(0, 2, 1).reshape(-1)
    order = order[order >= 0]
    cls = np.full(len(lm), -1)
    listed = lm != 0
    cls[listed] = np.array([0, 1, 2, 3])[np.argmax((lm[listed, None] >> np.arange(4)) & 1, axis=1)]
    return levels, lm, cls, order


def tiles_of(sample_list):
    nt = (len(sample_list) + TP - 1) // TP
    t = np.full(nt * TP, -1, np.int64)
    t[:len(sample_list)] = sample_list
    return t.reshape(nt, TP)


def distinct_per_group(corners):
    """corners (G, K) with -1 = none -> number of distinct ids per group"""
    s = np.sort(corners, axis=1)
    new = np.ones_like(s, bool)
    new[:, 1:] = s[:, 1:] != s[:, :-1]
    return (new & (s >= 0)).sum(1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--size", type=int, default=512, help="image side (c2: 512)")
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--nv", type=int, default=64, help="staged voxels per half tile and coarse level")
    ap.add_argument("--nv-fine", type=int, default=128, help="staged voxels per half tile and fine level")
    ap.add_argument("--sms", type=int, default=132)
    args = ap.parse_args()
    levels, lm, cls, order = replay(args.size, args.samples)
    per_class = [tiles_of(order[cls[order] == c]) for c in range(4)]
    n_tiles = sum(len(t) for t in per_class)
    print("synth-313, %dx%d, %d samples: %d listed samples, %d tiles (%.0f per CTA on %d SMs)"
          % (args.size, args.size, args.samples, int((cls >= 0).sum()), n_tiles, n_tiles / args.sms, args.sms))
    print("| level (channels, fp32 B/voxel) | corner bytes requested | distinct voxel bytes per tile | ratio | "
          "distinct voxels per half tile p50 / p99 / max | half tiles over the staging (%d coarse / %d fine voxels) |"
          % (args.nv, args.nv_fine))
    print("|---|---|---|---|---|---|")
    tot_req = tot_uniq = 0
    for lvl in (3, 2, 1, 0):
        L = levels[lvl]
        vb = L["C"] * 4
        req = uniq = 0
        halves = []
        for c, t in enumerate(per_class):
            if lvl < c or len(t) == 0:                                          # a class-c tile gathers levels 3 .. c
                continue
            valid = t >= 0
            s = np.where(valid, t, 0)
            occ = valid & (((lm[s] >> lvl) & 1) == 1)
            D, H, W = L["dims"]
            b = L["base"][s]
            corners = np.stack([b + (k & 1) + ((k >> 1) & 1) * W + (k >> 2) * W * H for k in range(8)], -1)
            corners = np.where(occ[..., None], corners, -1)                      # (tiles, 128, 8)
            req += int(occ.sum()) * 8 * vb
            uniq += int(distinct_per_group(corners.reshape(len(t), -1)).sum()) * vb
            hv = distinct_per_group(corners.reshape(len(t) * 2, -1))
            has_rows = valid.reshape(len(t) * 2, HALF).any(1)
            halves.append(hv[has_rows])
        h = np.concatenate(halves) if halves else np.zeros(1, np.int64)
        over = "%.2f %%" % (100.0 * (h > (args.nv if lvl >= 2 else args.nv_fine)).mean())
        print("| %d (%d ch, %d B; %.1f MB) | %.1f GB | %.2f GB | %.1fx | %d / %d / %d | %s |"
              % (lvl, L["C"], vb, np.prod(L["dims"]) * vb / 1e6, req / 1e9, uniq / 1e9, req / max(1, uniq),
                 np.percentile(h, 50), np.percentile(h, 99), h.max(), over))
        tot_req += req
        tot_uniq += uniq
    print("| all | %.1f GB | %.2f GB | %.0fx | | |" % (tot_req / 1e9, tot_uniq / 1e9, tot_req / max(1, tot_uniq)))


if __name__ == "__main__":
    main()
