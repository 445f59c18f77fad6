"""Diagnostics (GPU): per-role timeline of CTA 0 of the tensor-core render kernel, from the clock64 trace
the kernel writes when nb_render_args.trace is set.  Usage: python tools/trace_timeline.py [precision] [first_tile] [n_tiles]"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

# role 0: the row / per-point-tile warps (thread 32), 1 / 2: the two consumer warpgroups (threads 128 / 256), 3: the weight
# loader (thread 0)
PROD = {1: "tile begin", 30: "next tile's rows loaded", 31: "L2 done seen", 32: "per-point tile written"}
MMA = {1: "tile begin", 20: "L0 retired", 21: "L1 retired", 22: "L2 retired", 23: "L3 retired", 24: "raw stored"}
LOAD = {1: "first push of a tile issued", 2: "last push of a tile issued"}
VALUES = {50: "weight wait", 51: "row wait", 52: "per-point tile wait", 53: "gather coarse", 54: "gather fine"}   # cycles per tile
LAYERS = [(1, 20, "L0"), (20, 21, "L1"), (21, 22, "L2"), (22, 23, "L3"), (23, 24, "head")]


def main():
    prec = sys.argv[1] if len(sys.argv) > 1 else "tc_fp16x3"
    firsts = [int(v) for v in sys.argv[2].split(",")] if len(sys.argv) > 2 else [6]
    ntile = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    import gpu_utils as G
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    net, ren = G.make_net_and_renderer(scene)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.render_precision, cfg.render_volume_dtype = 64, 0.0, False, prec, "auto"
    cfg.render_skip_empty = not (len(sys.argv) > 4 and sys.argv[4] == "dense")
    net.eval()
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    sp = ren.prepare_sp_input(batch)
    vol = net.encode_sparse_voxels(sp)
    trace = torch.zeros(4 * 4096, dtype=torch.int64, device="cuda")
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    for _ in range(2):
        trace.zero_()
        ren.stats.zero_()
        with torch.no_grad():
            ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp, trace=trace)
    torch.cuda.synchronize()
    staged, direct = int(ren.stats[5]), int(ren.stats[6])
    print("coarse-level half tiles (levels 3 and 2, all CTAs): %d staged, %d direct (%.2f%% direct)"
          % (staged, direct, 100.0 * direct / max(1, staged + direct)))
    print("fine-level half tiles (levels 1 and 0, all CTAs): %d direct" % int(ren.stats[7]))
    t = trace.cpu().view(4, 4096)
    roles = [("PROD", PROD, None, 1), ("MMA0", MMA, None, 1), ("MMA1", MMA, None, 1), ("LOAD", LOAD, None, 1)]
    per_tile = {}                                            # (role, tile) -> {code: clock or value}
    events = []
    for r, (name, names, _, begin_code) in enumerate(roles):
        tile = -1
        for v in t[r].tolist():
            if v == 0:
                break
            code, clk = (v >> 48) & 0xFFFF, v & 0xFFFFFFFFFFFF
            if code == begin_code:
                tile += 1
            per_tile.setdefault((name, tile), {})[code] = clk
            if code in VALUES:
                continue
            events.append((clk, name, tile, names.get(code, str(code))))
    events.sort()
    for first in firsts:
        sel = [e for e in events if first <= e[2] < first + ntile]
        if not sel:
            continue
        t0 = sel[0][0]
        last = {}
        print("---- tiles %d..%d of CTA 0" % (first, first + ntile - 1))
        for clk, name, tile, what in sel:
            d = clk - last.get(name, clk)
            last[name] = clk
            print("%9d  (+%6d)  %-5s tile %-3d %s" % (clk - t0, d, name, tile, what))
    # per-tile summary of the consumer warpgroups: cycles per layer, cycles waited on weights / rows / the per-point tile, and
    # cycles spent gathering layer 0's features
    for name in ("MMA0", "MMA1"):
        tiles = [d for (r, _), d in sorted(per_tile.items()) if r == name and all(c in d for c in (1, 20, 21, 22, 23, 24, 50))]
        if len(tiles) < 2:
            continue
        tiles = tiles[1:]                                    # the first tile includes the pipeline fill
        row = ["%s %.0f" % (lbl, sum(d[b] - d[a] for d in tiles) / len(tiles)) for a, b, lbl in LAYERS]
        nxt = [b[1] - a[1] for a, b in zip(tiles[:-1], tiles[1:])]
        print("%s, mean over %d tiles (cycles): %s | tile period %.0f" % (name, len(tiles), "  ".join(row), sum(nxt) / max(1, len(nxt))))
        print("    per tile: " + "  ".join("%s %.0f" % (lbl, sum(d.get(c, 0) for d in tiles) / len(tiles)) for c, lbl in VALUES.items()))


if __name__ == "__main__":
    main()
