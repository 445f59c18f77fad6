"""Benchmark (GPU) of the mesh renderer (if_mesh_renderer) on the full-size synth-313 frame: density on the 5 mm world grid
(170x325x146) where it is inside the synthetic mask views, cube, marching cubes at --mesh-th.  One step = one frame, split
into its steps with CUDA events after warm-up.  Prints one JSON line with the split, the density kernel's FP32 rate, the
marching-cubes bytes/s, and the card's name and power limit read in the same run.  Writes nothing.

--density-precision picks cfg.density_precision (fp32, the default, or the tensor-core tc_fp16x3 / tc_fp16); --ab alternates
fp32 and tc_fp16x3 step by step in one process and reports the density ms of both arms.  For a tensor-core arm it also
reports the points listed for the decoder and skipped (stats[1]) and the algorithmic rate on the evaluated points only:
fc_0 (minus the layer-0 K-steps the tile's class skipped, as bench.py counts them for rays) + fc_1 + fc_2 + alpha_fc.

--from-masks compares, in one process and alternating frame by frame, the two ways the renderer gets its grid: (a) the
upstream data path, the world grid and its mask-view test on this host (mesh_case.mesh_grid + mesh_inside, numpy, as the
reference's mesh dataset builds them), the copy of `pts` / `inside` to the device and the render; (b) the copy of the
mask views and cameras to the device and the render, which builds the grid's axes on the host and its test on the device
(nb_mesh_inside).  4 synthetic 1024 x 1024 mask views; medians per frame of each step, the nb_mesh_inside kernel time
from CUDA events over back-to-back launches, and whether the two cubes are identical.  With --monocular the frame is the
People-Snapshot one instead (tools/mesh_mono_case.py, the monocular mesh dataset's bounds): one 540 x 540 mask view (a 1080 x
1080 frame at ratio 0.5) with the dataset's float64 camera, so (a) projects the grid in float64 numpy and (b) runs
nb_mesh_inside_f64.

--vis measures `run.py --type visualize` with `vis_mesh True` per frame, render + visualize, alternating two paths frame by
frame in one process: (a) `mesh_output: 'host'` and upstream's visualize body restated (`os.system('mkdir -p')`,
`mesh.export(path)` on the loop thread); (b) `mesh_output: 'device'` and the drop-in lib/visualizers/if_nerf_mesh.py.  It
reports the median ms per frame, each path's loop total in a loop of its own (the drop-in's final flush() included), the
nb_mesh_ply kernel alone (CUDA events over back-to-back launches) and its bytes/s, whether (a) and (b) wrote identical
files, and the card's name, power limit and SM clock read in the same run.  Files go to a temporary directory.

Usage: python tools/bench_mesh.py [--steps 5] [--warmup 3] [--mesh-th 10] [--density-precision P | --ab | --from-masks [--monocular] | --vis]
(upstream's default mesh_th = 50 lies above the synthetic body's sigma, p95 ~ 30, and would give an empty mesh)"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

FLOP_PER_POINT_DENSITY = 442880         # fc_0 + fc_1 + fc_2 + alpha_fc: 2 x (352*256 + 2*256*256 + 256) MAC per point
FLOP_L0_PER_KSTEP = 2 * 16 * 256        # one layer-0 K-step (16 of fc_0's 352 inputs), per point
FP32_TFLOPS_DATASHEET = 67.0             # H100 SXM data sheet, dense FP32 (700 W card)
HBM_TBS_DATASHEET = 3.35                 # H100 SXM data sheet, HBM3
PAD = 10


def card_info(dev):
    """Card name, power limit and SM clock, read in the same run as the measurement."""
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "sm_clock_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                              str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
        info["sm_clock_mhz"] = float(out.splitlines()[0])
    except Exception:
        pass
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev.index or 0)
        info["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:
        try:
            out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                                  str(dev.index or 0)], capture_output=True, text=True, timeout=30).stdout.strip()
            info["power_limit_w"] = float(out.splitlines()[0])
        except Exception:
            pass
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mesh-th", type=float, default=10.0, help="isovalue (cfg.mesh_th)")
    ap.add_argument("--density-precision", choices=("fp32", "tc_fp16x3", "tc_fp16"), default="fp32")
    ap.add_argument("--ab", action="store_true", help="alternate fp32 and tc_fp16x3 density steps in one process")
    ap.add_argument("--from-masks", action="store_true",
                    help="compare the host-built grid / inside (upstream's data path) with the device-built one")
    ap.add_argument("--monocular", action="store_true",
                    help="with --from-masks: the People-Snapshot frame (one view, float64 camera) instead of the 4-view one")
    ap.add_argument("--vis", action="store_true",
                    help="render + visualize per frame: host mode and upstream's visualize body against device mode and "
                         "the drop-in visualizer")
    args = ap.parse_args()
    if args.monocular and not args.from_masks:
        ap.error("--monocular goes with --from-masks")
    if args.from_masks:
        return from_masks(args)
    if args.vis:
        return vis(args)
    arms = ("fp32", "tc_fp16x3") if args.ab else (args.density_precision,)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device")
    from oracle import mesh_case
    from neuralbody_b200 import mcubes
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import make_network, load_source
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scene, _, batch = mesh_case.build_case("mesh_full")
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.voxel_size = list(scene["voxel_size"])
    cfg.mesh_th = float(args.mesh_th)
    net = make_network(cfg)
    net.load_state_dict(scene["weights"], strict=False)
    net = net.to(dev).eval()
    net.set_feature_volume([v.to(dev) for v in scene["volumes"]])
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")
    ren = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", path).Renderer(net)
    bd = {k: v.to(dev) for k, v in batch.items()}

    stats = torch.zeros(8, dtype=torch.int64, device=dev)

    def frame(arm):
        """Renderer.render (density_cube + marching cubes + copies) step by step, events between the steps."""
        cfg.density_precision = arm
        if getattr(net, "_density_renderer", None) is not None:
            net._density_renderer.stats = stats
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
        with torch.no_grad():
            ev[0].record()
            inside = bd["inside"][0].bool()
            wpts = bd["pts"][0][inside][None]
            sp = ren.prepare_sp_input(bd)
            fv = net.encode_sparse_voxels(sp)
            ev[1].record()
            alpha = net.calculate_density(wpts, fv, sp)
            ev[2].record()
            cube = torch.zeros(tuple(s + 2 * PAD for s in inside.shape), dtype=torch.float32, device=dev)
            cube[PAD:-PAD, PAD:-PAD, PAD:-PAD][inside] = alpha[0, :, 0]
            ev[3].record()
            verts, tris = mcubes.marching_cubes(cube, cfg.mesh_th)
            ev[4].record()
            mesh = mcubes.make_mesh(verts.cpu().numpy(), tris.cpu().numpy())
            ev[5].record()
            cube_host = cube.cpu().numpy().astype(np.float64)
            ev[6].record()
        return ev, int(wpts.shape[1]), mesh, cube_host

    for _ in range(args.warmup):
        for arm in arms:
            frame(arm)
    torch.cuda.synchronize(dev)
    rows = {arm: [] for arm in arms}
    arm_stats = {arm: [] for arm in arms}
    cubes = {}
    for _ in range(args.steps):
        for arm in arms:
            stats.zero_()
            ev, n_in, mesh, cube_host = frame(arm)
            torch.cuda.synchronize(dev)
            rows[arm].append([ev[i].elapsed_time(ev[i + 1]) for i in range(6)])
            arm_stats[arm].append([int(v) for v in stats.tolist()])
            cubes[arm] = cube_host
    density = {}
    for arm in arms:
        ms = float(np.median([r[1] for r in rows[arm]]))
        d = {"density_ms_median": ms, "density_ms_all": [r[1] for r in rows[arm]]}
        st = arm_stats[arm][-1]
        if arm == "fp32":
            d["tflops_fp32_kernel"] = FLOP_PER_POINT_DENSITY * n_in / (ms * 1e-3) / 1e12
        else:
            listed = st[1]
            l0 = st[4] / max(1, st[0])                       # layer-0 K-steps per executed tile (22 = all of fc_0)
            flop_pt = FLOP_PER_POINT_DENSITY - (22.0 - l0) * FLOP_L0_PER_KSTEP
            d.update({"points": n_in, "listed": listed, "skipped": n_in - listed, "evaluated_fraction": listed / max(1, n_in),
                      "layer0_ksteps_per_tile": l0, "flop_per_evaluated_point": flop_pt,
                      "decoder_kernel_ms": st[2] * 1e-6 / max(1, st[3]),
                      "tflops_evaluated_points": listed * flop_pt / (ms * 1e-3) / 1e12})
        density[arm] = d
    if args.ab:
        density["max_abs_cube_diff_vs_fp32"] = float(np.abs(cubes["tc_fp16x3"] - cubes["fp32"]).max())
    arm = arms[-1]                                         # the split, the public call and the mesh below: the last arm
    cfg.density_precision = arm
    rows = rows[arm]
    # the public call, whole (cube copy included); it must give the same result as the split steps
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        ren.render(bd)
        torch.cuda.synchronize(dev)
        t0.record()
        for _ in range(args.steps):
            out = ren.render(bd)
        t1.record()
        torch.cuda.synchronize(dev)
    render_ms = t0.elapsed_time(t1) / args.steps
    assert np.array_equal(np.asarray(out["mesh"].faces), np.asarray(mesh.faces)) and np.array_equal(out["cube"], cube_host)
    med = [float(np.median([r[i] for r in rows])) for i in range(6)]
    names = ("prepare_ms", "density_ms", "scatter_ms", "marching_cubes_ms", "mesh_to_host_ms", "cube_to_host_ms")
    split = dict(zip(names, med))
    excl_cube = sum(med[:5])
    nx, ny, nz = cube_host.shape
    n_pts = nx * ny * nz
    n_v, n_f = len(mesh.vertices), len(mesh.faces)
    # bytes the marching-cubes kernels move as written: count (grid 4 B read, code 2 B write per point), two scans
    # (code 2 B read, offset 4 B write each), emit (code + grid + two offsets read) + 24 B per vertex and per triangle
    mc_bytes = n_pts * (6 + 2 * 6 + 2 + 4 + 8) + 24 * (n_v + n_f)
    mc_gbs = mc_bytes / (split["marching_cubes_ms"] * 1e-3) / 1e9
    dens_tflops = FLOP_PER_POINT_DENSITY * n_in / (split["density_ms"] * 1e-3) / 1e12
    line = {
        "metric": "mesh_frame_ms_excl_cube_copy", "value": excl_cube, "unit": "ms", "higher_is_better": False,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
        "config": {"workload": "mesh renderer (if_mesh_renderer) on the full-size synth-313 frame: 5 mm world grid %s, inside "
                               "from 4 synthetic 256x256 mask views, cube padded to %s, marching cubes at mesh_th = %g"
                               % (tuple(batch["inside"].shape[1:]), (nx, ny, nz), cfg.mesh_th),
                   "grid_points": int(np.prod(batch["inside"].shape)), "padded_points": n_pts},
        "inside_points": n_in, "vertices": n_v, "triangles": n_f,
        "split_ms_median": split, "render_ms_excl_cube_copy": excl_cube, "render_call_ms": render_ms,
        "density": {"flop_per_point": FLOP_PER_POINT_DENSITY, "tflops": dens_tflops,
                    "fraction_of_fp32_datasheet": dens_tflops / FP32_TFLOPS_DATASHEET,
                    "datasheet": "67 TFLOP/s dense FP32, H100 SXM at 700 W (not a reached figure)"} if arm == "fp32" else
                   {"see": "density_arms"},
        "marching_cubes": {"bytes_as_written": mc_bytes, "gbs": mc_gbs, "fraction_of_hbm_datasheet": mc_gbs / (HBM_TBS_DATASHEET * 1e3),
                           "note": "includes the one host sync between count and emit and the launch gaps"},
        "density_precision": arm, "density_arms": density,
        "card": card_info(dev),
    }
    print(json.dumps(line))


def from_masks(args):
    """--from-masks: arm (a) upstream's data path (host grid + host inside + H2D of pts / inside + render), arm (b) H2D of
    the mask views and cameras + render from them; one JSON line."""
    import ctypes as C
    import time
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device")
    from oracle import mesh_case, synth
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import make_network, load_source
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    if args.monocular:
        from tools import mesh_mono_case as MM
        scene, pkl, _, _ = MM.build_case("mono_full")
        K = MM.get_camera(pkl)["K"].copy()
        K[:2] = K[:2] * MM.RATIO                                     # the dataset's K after its resize, float64
        msk = MM.silhouette(scene, K, 540, 540, 2)
        Ks, Rs, Ts, msks = K[None], np.eye(3)[None], np.zeros((1, 3, 1)), msk[None]
        masks = {"RT": torch.from_numpy(np.concatenate([Rs, Ts], axis=2))[None], "Ks": torch.from_numpy(Ks)[None],
                 "msks": torch.from_numpy(msks)[None]}
        host_inside = lambda pts: MM.mesh_inside_f64(pts, K, Rs[0], Ts[0], msk)    # noqa: E731
    else:
        scene = synth.make_scene(**mesh_case.CASES["mesh_full"][0])
        masks = synth.make_mask_views(scene, nv=4, H=1024, W=1024, radius=12)
        Ks, Rs, Ts, msks = mesh_case._views(masks)
        host_inside = lambda pts: mesh_case.mesh_inside(pts, Ks, Rs, Ts, msks)    # noqa: E731
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.voxel_size = list(scene["voxel_size"])
    cfg.mesh_th = float(args.mesh_th)
    cfg.density_precision = args.density_precision
    net = make_network(cfg)
    net.load_state_dict(scene["weights"], strict=False)
    net = net.to(dev).eval()
    net.set_feature_volume([v.to(dev) for v in scene["volumes"]])
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")
    mod = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", path)
    ren = mod.Renderer(net)
    frame = {k: scene[k].to(dev) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    cb = scene["can_bounds"][0].numpy()

    def sync_ms(t0):
        torch.cuda.synchronize(dev)
        return (time.perf_counter() - t0) * 1e3

    def arm_host():
        t = time.perf_counter()
        pts = mesh_case.mesh_grid(cb, scene["voxel_size"])
        t_grid = (time.perf_counter() - t) * 1e3
        t = time.perf_counter()
        inside = host_inside(pts)
        t_inside = (time.perf_counter() - t) * 1e3
        t = time.perf_counter()
        b = dict(frame, pts=torch.from_numpy(pts)[None].to(dev), inside=torch.from_numpy(inside)[None].to(dev))
        t_h2d = sync_ms(t)
        t = time.perf_counter()
        with torch.no_grad():
            out = ren.render(b)
        t_render = sync_ms(t)
        return {"grid_host_ms": t_grid, "inside_host_ms": t_inside, "h2d_ms": t_h2d, "render_ms": t_render,
                "h2d_bytes": pts.nbytes + inside.nbytes}, out, int(inside.astype(bool).sum())

    def arm_device():
        t = time.perf_counter()
        b = dict(frame, wbounds=scene["can_bounds"].to(dev), RT=masks["RT"].to(dev), Ks=masks["Ks"].to(dev),
                 msks=masks["msks"].to(dev))
        t_h2d = sync_ms(t)
        t = time.perf_counter()
        with torch.no_grad():
            wpts, _ = ren.grid_from_masks(b)
        t_grid = sync_ms(t)
        t = time.perf_counter()
        with torch.no_grad():
            out = ren.render(b)
        t_render = sync_ms(t)
        nbytes = sum(int(b[k].numel() * b[k].element_size()) for k in mod.MASK_KEYS)
        return {"h2d_ms": t_h2d, "grid_from_masks_ms": t_grid, "render_ms": t_render, "h2d_bytes": nbytes}, out, int(wpts.shape[1])

    for _ in range(args.warmup):
        arm_host(); arm_device()
    rows = {"a_host_grid": [], "b_device_grid": []}
    for _ in range(args.steps):
        ra, out_a, n_a = arm_host()
        rb, out_b, n_b = arm_device()
        rows["a_host_grid"].append(ra)
        rows["b_device_grid"].append(rb)
    med = {arm: {k: float(np.median([r[k] for r in rs])) for k in rs[0]} for arm, rs in rows.items()}
    med["a_host_grid"]["frame_ms"] = sum(med["a_host_grid"][k] for k in ("grid_host_ms", "inside_host_ms", "h2d_ms", "render_ms"))
    med["b_device_grid"]["frame_ms"] = sum(med["b_device_grid"][k] for k in ("h2d_ms", "render_ms"))

    # nb_mesh_inside alone: back-to-back launches between two CUDA events
    axes = [torch.from_numpy(a).to(dev) for a in mod.world_axes(cb, scene["voxel_size"])]
    m, rt = masks["msks"][0].to(dev).contiguous(), masks["RT"][0].to(dev).contiguous()
    ks = masks["Ks"][0].to(dev).contiguous()
    inside = torch.empty(tuple(len(a) for a in axes), dtype=torch.uint8, device=dev)
    a = capi.nb_mesh_inside_args()
    a.x, a.y, a.z = (t.data_ptr() for t in axes)
    a.nx, a.ny, a.nz = inside.shape
    a.msks, a.inside = m.data_ptr(), inside.data_ptr()
    a.nv, a.H, a.W = (int(s) for s in m.shape)
    lib, stream = capi.load(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    if args.monocular:
        entry = "nb_mesh_inside_f64"
        launch = lambda: lib.nb_mesh_inside_f64(C.byref(a), rt.data_ptr(), ks.data_ptr(), stream)    # noqa: E731
    else:
        entry = "nb_mesh_inside"
        a.RT, a.Ks = rt.data_ptr(), ks.data_ptr()
        launch = lambda: lib.nb_mesh_inside(C.byref(a), stream)    # noqa: E731
    launches = 200
    for _ in range(20):
        capi.check(launch(), entry)
    kernel_ms = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            launch()
        e1.record()
        torch.cuda.synchronize(dev)
        kernel_ms.append(e0.elapsed_time(e1) / launches)
    n_pts = inside.numel()
    line = {
        "metric": "mesh_frame_ms_from_masks", "value": med["b_device_grid"]["frame_ms"], "unit": "ms", "higher_is_better": False,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
        "config": {"workload": "mesh renderer on the full-size synth-313 frame: 5 mm world grid %s (%d points), %s, "
                               "density %s, mesh_th = %g; render = the whole Renderer.render call (cube copy to the host "
                               "included)" % (tuple(inside.shape), n_pts, "one synthetic 540x540 People-Snapshot mask view, "
                                              "float64 camera" if args.monocular else "4 synthetic 1024x1024 mask views",
                                              args.density_precision, cfg.mesh_th)},
        "inside_points": {"a": n_a, "b": n_b},
        "cubes_identical": bool(out_a["cube"].shape == out_b["cube"].shape and np.array_equal(out_a["cube"], out_b["cube"])),
        "meshes_identical": bool(np.array_equal(np.asarray(out_a["mesh"].faces), np.asarray(out_b["mesh"].faces)) and
                                 np.array_equal(np.asarray(out_a["mesh"].vertices), np.asarray(out_b["mesh"].vertices))),
        "median_ms": med, "speedup_frame": med["a_host_grid"]["frame_ms"] / med["b_device_grid"]["frame_ms"],
        "kernel": entry,
        "nb_mesh_inside_kernel_ms": {"median": float(np.median(kernel_ms)), "all": kernel_ms, "launches_per_sample": launches,
                                     "gpoints_per_s": n_pts / (float(np.median(kernel_ms)) * 1e-3) / 1e9},
        "host_cpus": os.cpu_count(), "numpy": np.__version__,
        "card": card_info(dev),
    }
    print(json.dumps(line))


def vis(args):
    """--vis: arm (a) host mode + upstream's visualize body, arm (b) device mode + the drop-in visualizer; one JSON line."""
    import contextlib
    import ctypes as C
    import filecmp
    import tempfile
    import time
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device")
    from oracle import mesh_case
    from neuralbody_b200 import capi, mcubes
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import make_network, load_source
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scene, _, batch = mesh_case.build_case("mesh_full")
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.voxel_size = list(scene["voxel_size"])
    cfg.mesh_th = float(args.mesh_th)
    cfg.density_precision = args.density_precision
    net = make_network(cfg)
    net.load_state_dict(scene["weights"], strict=False)
    net = net.to(dev).eval()
    net.set_feature_volume([v.to(dev) for v in scene["volumes"]])
    lib_dir = os.path.join(ROOT, "neuralbody_b200", "lib")
    ren = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer",
                      os.path.join(lib_dir, "networks", "renderer", "if_mesh_renderer.py")).Renderer(net)
    vis_mod = load_source("neuralbody_b200.lib.visualizers.if_nerf_mesh", os.path.join(lib_dir, "visualizers", "if_nerf_mesh.py"))
    bd = {k: v.to(dev) for k, v in batch.items()}
    tmp = tempfile.TemporaryDirectory()
    dirs = {"a": os.path.join(tmp.name, "a"), "b": os.path.join(tmp.name, "b")}

    def upstream_visualize(output, b):
        """lib/visualizers/if_nerf_mesh.py:28-36 of the reference, restated."""
        mesh = output['mesh']
        result_dir = os.path.join(cfg.result_dir, 'mesh')
        os.system('mkdir -p {}'.format(result_dir))
        i = b['frame_index'].item()
        mesh.export(os.path.join(result_dir, '{:04d}.ply'.format(i)))

    cfg.result_dir = dirs["b"]
    with contextlib.redirect_stdout(sys.stderr):             # its "results are saved at" line: stdout keeps the JSON
        drop_in = vis_mod.Visualizer()

    def frame(arm, i):
        """One frame of `arm` -> host ms from the render call to visualize()'s return."""
        b = dict(bd, frame_index=torch.tensor([i], device=dev))
        cfg.mesh_output = "host" if arm == "a" else "device"
        cfg.result_dir = dirs[arm]
        t = time.perf_counter()
        with torch.no_grad():
            out = ren.render(b)
        (upstream_visualize if arm == "a" else drop_in.visualize)(out, b)
        return (time.perf_counter() - t) * 1e3

    for i in range(args.warmup):
        frame("a", i)
        frame("b", i)
    drop_in.flush()
    torch.cuda.synchronize(dev)
    rows = {"a": [], "b": []}
    for i in range(args.steps):
        for arm in ("a", "b"):
            rows[arm].append(frame(arm, args.warmup + i))
    t = time.perf_counter()
    drop_in.flush()
    flush_ms = (time.perf_counter() - t) * 1e3
    names = ["%04d.ply" % i for i in range(args.steps + args.warmup)]
    identical = all(filecmp.cmp(os.path.join(dirs["a"], "mesh", n), os.path.join(dirs["b"], "mesh", n), shallow=False)
                    for n in names)
    # each path's loop total in a loop of its own, the drop-in's final flush() included
    loops = {}
    for arm in ("a", "b"):
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        for i in range(args.steps):
            frame(arm, i)
        if arm == "b":
            drop_in.flush()
        loops[arm] = (time.perf_counter() - t) * 1e3

    # nb_mesh_ply alone on this frame's mesh: back-to-back launches between two CUDA events
    cfg.mesh_output = "device"
    with torch.no_grad():
        mesh = ren.render(dict(bd, frame_index=torch.tensor([0], device=dev)))["mesh"]
    out = torch.empty(capi.NB_MESH_PLY_BODY_OFFSET + mesh.body_bytes(), dtype=torch.uint8, device=dev)
    a = capi.nb_mesh_ply_args()
    a.nv, a.nf, a.vertices, a.faces = mesh.nv, mesh.nf, mesh.vertices.data_ptr(), mesh.faces.data_ptr()
    a.out, a.out_bytes = out.data_ptr(), out.numel()
    lib, stream = capi.load(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    launches = 200
    for _ in range(20):
        capi.check(lib.nb_mesh_ply(C.byref(a), stream), "nb_mesh_ply")
    kernel_ms = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            lib.nb_mesh_ply(C.byref(a), stream)
        e1.record()
        torch.cuda.synchronize(dev)
        kernel_ms.append(e0.elapsed_time(e1) / launches)
    k_ms = float(np.median(kernel_ms))
    moved = 24 * mesh.nv + 24 * mesh.nf + mesh.body_bytes()      # vertices and faces read once, the body written once
    med = {arm: float(np.median(r)) for arm, r in rows.items()}
    line = {
        "metric": "mesh_vis_frame_ms", "value": med["b"], "unit": "ms", "higher_is_better": False,
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "data": "synthetic",
        "config": {"workload": "run.py --type visualize with vis_mesh True on the full-size synth-313 frame: render (5 mm "
                               "world grid %s, density %s, marching cubes at mesh_th = %g) + visualize, one PLY per frame"
                               % (tuple(batch["inside"].shape[1:]), args.density_precision, cfg.mesh_th),
                   "a": "mesh_output 'host' + upstream's visualize body (os.system mkdir -p, mesh.export on the loop)",
                   "b": "mesh_output 'device' + lib/visualizers/if_nerf_mesh.py (nb_mesh_ply, pinned copy, writer thread)"},
        "vertices": mesh.nv, "triangles": mesh.nf, "ply_bytes": len(mcubes.ply_header(mesh.nv, mesh.nf)) + mesh.body_bytes(),
        "frame_ms_median": med, "frame_ms_all": rows, "speedup_frame": med["a"] / med["b"],
        "b_final_flush_ms": flush_ms,
        "loop_total_ms": {"a": loops["a"], "b_incl_flush": loops["b"], "frames": args.steps},
        "files_identical": bool(identical), "files_compared": len(names),
        "nb_mesh_ply_kernel": {"ms_median": k_ms, "ms_all": kernel_ms, "launches_per_sample": launches,
                               "bytes_moved": moved, "tbs": moved / (k_ms * 1e-3) / 1e12,
                               "fraction_of_hbm_datasheet": moved / (k_ms * 1e-3) / 1e12 / HBM_TBS_DATASHEET},
        "host_cpus": os.cpu_count(),
        "card": card_info(dev),
    }
    tmp.cleanup()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
