"""GPU: every row of the tensor-core decoder against an emulation of its own roundings (oracle/tc_decoder_model.py), on tiles
built to hit each staging, class and tail edge (oracle/decoder_tiles.py), with the decoder's counters proving each edge ran.

Per row: (a) the emulation within a measured tolerance, (b) the float64 oracle at the project's gates, (c) a fixed set of
probe points gives the same sigma bits in every tile it is decoded in.  The density cases run through
nb_decode_density_list (Renderer.calculate_density); the render rows through nb_render_fwd with caller depths and want_raw
on the golden scenes.  Each case runs for both tensor-core precisions, fp32 and fp16 volume blobs (the volumes are
fp16-representable, so both blobs hold the same numbers) and skipping on and off."""
import pytest
import torch

import gpu_utils as G
from conftest import golden_case
from oracle import decoder_tiles as T
from oracle import neuralbody_oracle as O
from oracle import synth
from oracle import tc_decoder_model as M
from neuralbody_b200.lib.config import cfg

pytestmark = pytest.mark.gpu

PASSES = {"tc_fp16x3": 3, "tc_fp16": 1}
# |GPU - emulation| bounds on raw sigma and the rgb logits per mode: the worst row (TOL_EMU) and the median row (TOL_MED), at
# about three times the values measured over every case and scene here on an NVIDIA H100 80GB HBM3 (700 W power limit), with
# the emulation accumulating each K-step into a float32 accumulator rounded toward zero (ACC = "rz"):
#   worst   sigma 5.3e-5 (3-pass) / 8.6e-3 (1-pass), logits 4.6e-4 / 4.6e-4
#   median  sigma 1.3e-5 / 5.2e-6,                  logits 2.4e-7 / 2.4e-7
# With a float64 accumulator instead the 3-pass sigma gap was 1.4e-4 worst and 8.3e-5 median, as large as the gap to the
# float64 oracle: the wgmma accumulation, not a rounding of the operands, held the rest of it.  The worst 3-pass logits and
# 1-pass rows come from rows where that accumulation flips an fp16 rounding (h2, or a 1-pass operand); the medians bound
# the rest, which is where a systematic one-ulp error (an operand rounded the wrong way) shows.
TOL_EMU = {("sigma", 3): 1.5e-4, ("sigma", 1): 3e-2, ("logit", 3): 1.5e-3, ("logit", 1): 1.5e-3}
TOL_MED = {("sigma", 3): 4e-5, ("sigma", 1): 2e-5, ("logit", 3): 1e-6, ("logit", 1): 1e-6}
GATE_SIGMA = {3: 5e-4, 1: 8e-2}           # vs the float64 oracle: test_density_tc_gpu.py's gates
GATE_LOGIT = {3: 2e-2, 1: 1e-1}
GATE_MAP = {3: 1e-3, 1: 3e-3}
WRAP_POINTS = 80037                       # ~64 K listed rows = 500 tiles > 3 x 132 SMs: every persistent CTA runs at least 3

ACC = "rz"                                # the emulation's accumulation model (tc_decoder_model._accumulate)

_cache = {}


def _with(**kw):
    old = {k: (cfg[k] if k in cfg else None) for k in kw}
    for k, v in kw.items():
        cfg[k] = v
    return old


def _restore(old):
    for k, v in old.items():
        if v is None:
            if k in cfg:
                del cfg[k]
        else:
            cfg[k] = v


def _weights():
    return golden_case("eval_s64")[0]["weights"]


def _probe_group(where):
    """128 class-0 points with the probes at the head (beside local neighbours: staged on every level) or at the tail
    (beside random ones: direct on every level); tests/test_decoder_rows_cpu.py checks both paths."""
    p = T.probe_points()
    if where == "head":
        return torch.cat([p, T.local_points(0, 112, seed=21)])
    return torch.cat([T.random_points(0, 112, seed=22), p])


def _density_cases():
    lim = [T.limit_group(3, 64, 65), T.limit_group(2, 64, 65), T.limit_group(1, 128, 129), T.limit_group(0, 128, 129)]
    rnd = {c: T.random_points(c, 128, seed=30 + i) for i, c in enumerate((3, 2, 1, 0, "gap", "empty"))}
    edges = lim + T.groups_by_class(T.boundary_points()) + [rnd["empty"], rnd["gap"], _probe_group("head")]
    cases = {
        "edges": (edges, True),
        "all_classes": ([rnd[3], rnd[2], rnd[1], rnd[0], _probe_group("tail")], True),
        "classes_3_0": ([rnd[3], _probe_group("tail"), rnd[0]], True),
        "classes_2_1": ([rnd[2], rnd["gap"], rnd[1]], True),
    }
    for c in (3, 2, 1):
        cases["class_%d_alone" % c] = ([rnd[c], T.random_points(c, 128, seed=40 + c)], True)
    cases["class_0_alone"] = ([_probe_group("head"), rnd[0]], True)
    tail_pts = torch.cat([_probe_group("head"), rnd[3], rnd[1]])
    for n in (1, 63, 64, 65, 127, 128, 129, 255, 256, 257):
        cases["n%d" % n] = ([tail_pts[:n]], False)
    g = torch.Generator().manual_seed(50)
    mix = torch.cat([T.random_points(r, WRAP_POINTS // 5 + 1, seed=51 + i) for i, r in enumerate((3, 2, 1, 0, "empty"))])
    mix = mix[torch.randperm(mix.shape[0], generator=g)][:WRAP_POINTS - 16]
    cases["wrap"] = ([torch.cat([mix, T.probe_points()])], False)
    return cases


CASES = _density_cases()
CASE_NAMES = list(CASES) + ["batch3"]


def _frames(B):
    """B frames that differ in pose, latent code and volume values (same occupancy, so the same tiles)."""
    key = ("frames", B)
    if key not in _cache:
        fr = [T.frame(b) for b in range(B)]
        vols = [torch.cat(v) for v in zip(*[T.make_volumes(100 + b) for b in range(B)])]
        R = torch.stack([f[0] for f in fr])
        Th = torch.stack([f[1] for f in fr])
        bounds = torch.stack([f[2] for f in fr])
        li = torch.tensor([0, 7, 33][:B], dtype=torch.int64)
        _cache[key] = (R, Th, bounds, li, vols)
    return _cache[key]


def _renderer(vols):
    key = ("ren", id(vols))
    if key not in _cache:
        scene = {"weights": _weights(), "voxel_size": list(T.VOXEL), "volumes": vols}
        net, ren = G.make_net_and_renderer(scene)
        _cache[key] = (net, ren, [v.cuda() for v in vols])
    return _cache[key]


def _case(name):
    if name == "batch3":
        groups, aligned = CASES["edges"]
        return groups, aligned, 3
    groups, aligned = CASES[name]
    return groups, aligned, 1


def _emulation(name, passes):
    key = ("emu", name, passes)
    if key not in _cache:
        groups, _, B = _case(name)
        q0 = torch.cat(groups)
        R, Th, bounds, li, vols = _frames(B)
        out = []
        q0 = q0[_rows(name)]
        for b in range(B):
            w = T.world_points(q0, R[b], Th[b], bounds[b])
            out.append(M.decode_frame(_weights(), int(li[b]), w, [v[b] for v in vols], R[b], Th[b], bounds[b], T.VOXEL,
                                      T.OUT_SH, passes=passes, density=True, acc=ACC))
        _cache[key] = torch.stack(out)
    return _cache[key]


def _rows(name):
    """The rows the emulation restates: every 8th of the 80 K-point case, all of the others."""
    n = torch.cat(_case(name)[0]).shape[0]
    return torch.arange(0, n, 8 if name == "wrap" else 1)


def _oracle(name):
    key = ("oracle", name)
    if key not in _cache:
        groups, _, B = _case(name)
        q0 = torch.cat(groups)
        R, Th, bounds, li, vols = _frames(B)
        wpts = torch.stack([T.world_points(q0, R[b], Th[b], bounds[b]) for b in range(B)])
        sp = {"R": R.double(), "Th": Th.double(), "bounds": bounds.double(), "out_sh": list(T.OUT_SH)}
        w = {k: v.double() for k, v in _weights().items()}
        _cache[key] = O.calculate_density(w, wpts.double(), [v.double() for v in vols], sp, T.VOXEL)[..., 0]
    return _cache[key]


def _run_density(name, precision, vdtype, skip):
    groups, _, B = _case(name)
    q0 = torch.cat(groups)
    R, Th, bounds, li, vols = _frames(B)
    net, ren, fv = _renderer(vols)
    wpts = torch.stack([T.world_points(q0, R[b], Th[b], bounds[b]) for b in range(B)]).cuda()
    sp = {"R": R.cuda(), "Th": Th.cuda(), "bounds": bounds.cuda(), "out_sh": list(T.OUT_SH), "latent_index": li.cuda()}
    old = _with(density_precision=precision, render_skip_empty=skip, render_volume_dtype=vdtype)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    try:
        sigma = ren.calculate_density(wpts, fv, sp)[..., 0]
        torch.cuda.synchronize()
        stats = ren.stats.cpu().tolist()
    finally:
        ren.stats = None
        _restore(old)
    return sigma.cpu(), stats


@pytest.mark.parametrize("skip", [True, False], ids=["skip", "noskip"])
@pytest.mark.parametrize("vdtype", ["fp32", "fp16"])
@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
@pytest.mark.parametrize("name", CASE_NAMES)
def test_density_rows(name, precision, vdtype, skip):
    groups, aligned, B = _case(name)
    passes = PASSES[precision]
    sigma, stats = _run_density(name, precision, vdtype, skip)
    q0 = torch.cat(groups)
    # the counters the construction predicts; per frame, so B frames count B times
    if aligned:
        want = T.tile_stats(groups, skip)
        for k in (0, 1, 4, 5, 6, 7):
            assert stats[k] == B * want[k], (k, stats, want)
    else:
        want = T.stats_by_class(T.classes(q0, skip))
        for k in (0, 1, 4):
            assert stats[k] == B * want[k], (k, stats, want)
    emu, ora = _emulation(name, passes), _oracle(name)
    de = (sigma[:, _rows(name)] - emu).abs()
    d_emu, m_emu = float(de.max()), float(de.median())
    d_ora = float((sigma.double() - ora).abs().max())
    print("ROWS density %s %s %s %s: |gpu - emulation| max %.3e median %.3e, |gpu - oracle| %.3e, stats %s"
          % (name, precision, vdtype, "skip" if skip else "noskip", d_emu, m_emu, d_ora, stats))
    assert d_emu <= TOL_EMU[("sigma", passes)], d_emu
    assert m_emu <= TOL_MED[("sigma", passes)], m_emu
    assert d_ora <= GATE_SIGMA[passes], d_ora


def _probe_id(q):
    return tuple(float(v) for v in q)


def _probe_rows(q0, p):
    """Rows of q0 that hold a probe point."""
    pid = {_probe_id(r) for r in p}
    return torch.tensor([i for i in range(q0.shape[0]) if _probe_id(q0[i]) in pid], dtype=torch.long)


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_probes_are_bit_identical_in_every_context(precision):
    """nb_decode_density_list's contract: a point's sigma does not depend on its tile.  The 16 probes are decoded at the
    head of a tile whose halves are staged on every level ('edges', 'class_0_alone'), at the tail of one gathered directly
    on every level ('all_classes', 'classes_3_0'), in short tiles ('n1' .. 'n257'), among 80 K points ('wrap') and as frame 0
    of a three-frame call, each with both blobs and skipping on and off; every context must give the first one's bits."""
    p = T.probe_points()
    ref, seen = None, 0
    for name in ["edges", "class_0_alone", "all_classes", "classes_3_0", "wrap", "batch3"] + \
            ["n%d" % n for n in (1, 63, 64, 65, 127, 128, 129, 255, 256, 257)]:
        q0 = torch.cat(_case(name)[0])
        idx = _probe_rows(q0, p)
        for vdtype in ("fp32", "fp16"):
            for skip in (True, False):
                sigma, _ = _run_density(name, precision, vdtype, skip)
                got = {_probe_id(q0[r]): int(v) for r, v in zip(idx.tolist(), sigma[0, idx].contiguous().view(torch.int32).tolist())}
                if ref is None:
                    ref = got
                    assert len(ref) == p.shape[0]
                for k, v in got.items():
                    assert v == ref[k], (name, vdtype, skip, k)
                seen += len(got)
    assert seen > 40 * p.shape[0]


# ------------------------------------------------------------------------------------------------ render rows
RENDER_SCENES = ["designed", "designed_tail", "eval_s64", "batch2_s32", "train_jitter_white", "full_313"]
DESIGNED_TAIL_RAYS = 777                  # an odd ray count: the second block of 512 rays is cut in its fourth group


def _designed_groups():
    """Groups of the designed render view (each 128 points of one class, y < 40 so that the second sample, moved by one
    level-3 voxel along y, stays inside): the 64 / 65 and 128 / 129 limits, all four classes, the level gap, boundary
    cells and empty points, 4 groups per block of 512 rays."""
    lim = [T.limit_group(3, 64, 65), T.limit_group(2, 64, 65), T.limit_group(1, 128, 129), T.limit_group(0, 128, 129)]
    b = T.boundary_points()
    b = b[b[:, 1] < 40]
    rnd = [T.random_points(r, 128, seed=60 + i, ymax=40) for i, r in enumerate(("empty", "gap", 2, 0, 3))]
    groups = lim + rnd + T.groups_by_class(b)
    while len(groups) % 4:
        groups.append(T.random_points(1, 128, seed=70 + len(groups), ymax=40))
    return groups


def _designed_scene(name):
    R, Th, bounds, li, vols = _frames(1)
    groups = _designed_groups()
    o, d, z, _ = T.render_rays(groups, R[0], Th[0], bounds[0])
    n = o.shape[0] if name == "designed" else DESIGNED_TAIL_RAYS
    scene = {"ray_o": o[None, :n].contiguous(), "ray_d": d[None, :n].contiguous(), "near": z[None, :n, 0] - 0.1,
             "far": z[None, :n, 1] + 0.1, "R": R, "Th": Th, "bounds": bounds, "latent_index": li,
             "out_sh": torch.tensor([T.OUT_SH], dtype=torch.int32), "coord": torch.zeros((1, 1, 3), dtype=torch.int32),
             "volumes": vols, "weights": _weights(), "voxel_size": list(T.VOXEL)}
    return scene, z[None, :n].contiguous(), False


def _designed_stats(name, skip):
    """The render counters the designed view predicts: exact for whole blocks, by class for the cut one."""
    groups = _designed_groups()
    if name == "designed":
        return T.tile_stats(T.render_groups(groups), skip), (0, 1, 4, 5, 6, 7)
    _, _, _, q = T.render_rays(groups, *[t[0] for t in _frames(1)[:3]])
    return T.stats_by_class(T.classes(q[:DESIGNED_TAIL_RAYS].reshape(-1, 3), skip)), (0, 1, 4)


def _render_case(name):
    key = ("rscene", name)
    if key not in _cache and name.startswith("designed"):
        _cache[key] = _designed_scene(name)
    if key not in _cache:
        scene, rkw, _ = golden_case(name)
        if name == "full_313":
            scene = dict(scene)
            for k in ("ray_o", "ray_d", "near", "far"):
                scene[k] = scene[k][:, ::4].contiguous()
        scene = synth.rounded_scene(scene)
        S = rkw["n_samples"]
        t_rand = rkw.get("t_rand")
        if t_rand is not None and name == "full_313":
            t_rand = t_rand[:, ::4]
        _, z = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], S,
                                     rkw.get("perturb", 0.0), rkw.get("training", False), t_rand)
        _cache[key] = (scene, z.float().contiguous(), bool(rkw.get("white_bkgd", False)))
    return _cache[key]


def _render_reference(name, passes):
    key = ("rref", name, passes)
    if key not in _cache:
        scene, z, white = _render_case(name)
        B, n, S = z.shape
        sp = O.prepare_sp_input(scene)
        emu, ora = [], []
        w64 = {k: v.double() for k, v in scene["weights"].items()}
        for b in range(B):
            pts = M.sample_points_f32(scene["ray_o"][b], scene["ray_d"][b], z[b]).reshape(-1, 3)
            rd = scene["ray_d"][b][:, None].expand(n, S, 3).reshape(-1, 3)
            emu.append(M.decode_frame(scene["weights"], int(scene["latent_index"][b]), pts, [v[b] for v in scene["volumes"]],
                                      sp["R"][b], sp["Th"].reshape(B, 3)[b], sp["bounds"][b], scene["voxel_size"],
                                      sp["out_sh"], passes=passes, ray_d=rd, acc=ACC).reshape(n, S, 4))
        emu = torch.stack(emu)
        if passes == 3:
            vd = scene["ray_d"].double() / torch.norm(scene["ray_d"].double(), dim=2, keepdim=True)
            pts = M.sample_points_f32(scene["ray_o"].reshape(-1, 3), scene["ray_d"].reshape(-1, 3),
                                      z.reshape(B * n, S)).reshape(B, n * S, 3)
            vdx = vd[:, :, None].expand(B, n, S, 3).reshape(B, n * S, 3)
            sp64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sp.items()}
            raw = O.calculate_density_color(w64, pts.double(), vdx, [v.double() for v in scene["volumes"]], sp64,
                                            scene["voxel_size"]).reshape(B, n, S, 4)
            maps = O.raw2outputs(raw.reshape(B * n, S, 4), z.double().reshape(B * n, S),
                                 scene["ray_d"].double().reshape(-1, 3), white)
            _cache[("rora", name)] = (raw, {"rgb_map": maps[0].reshape(B, n, 3), "acc_map": maps[2].reshape(B, n),
                                            "depth_map": maps[4].reshape(B, n)})
        _cache[key] = emu
    if ("rora", name) not in _cache:
        _render_reference(name, 3)
    return _cache[key], _cache[("rora", name)]


@pytest.mark.parametrize("skip", [True, False], ids=["skip", "noskip"])
@pytest.mark.parametrize("vdtype", ["fp32", "fp16"])
@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
@pytest.mark.parametrize("name", RENDER_SCENES)
def test_render_rows(name, precision, vdtype, skip):
    scene, z, white = _render_case(name)
    passes = PASSES[precision]
    emu, (ora_raw, ora_maps) = _render_reference(name, passes)
    net, ren = G.make_net_and_renderer(scene)
    old = _with(N_samples=z.shape[-1], perturb=0.0, white_bkgd=white, raw_noise_std=0, render_precision=precision,
                render_volume_dtype=vdtype, render_skip_empty=skip)
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    try:
        sp = ren.prepare_sp_input(batch)
        with torch.no_grad():
            out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], net.encode_sparse_voxels(sp),
                                  sp, z_vals=z.cuda(), want_raw=True)
        torch.cuda.synchronize()
        stats = ren.stats.cpu().tolist()
    finally:
        ren.stats = None
        _restore(old)
    if name.startswith("designed"):
        want, keys = _designed_stats(name, skip)
        for k in keys:
            assert stats[k] == want[k], (k, stats, want)
    raw = out["raw"].cpu()
    # a skipped sample's record is (0, 0, 0, min(sigma_empty, 0)); compare the evaluated ones
    ev = ~(raw[..., :3] == 0).all(-1)
    if skip:
        assert 0 < int(ev.sum()) < ev.numel()
        assert bool((raw[..., 3][~ev] == raw[..., 3][~ev][0]).all())
    else:
        assert bool(ev.all())
    ds, dl = (raw[..., 3] - emu[..., 3])[ev].abs(), (raw[..., :3] - emu[..., :3])[ev].abs()
    d_sig, d_log, m_sig, m_log = float(ds.max()), float(dl.max()), float(ds.median()), float(dl.median())
    o_sig = float((raw[..., 3].double() - ora_raw[..., 3])[ev].abs().max())
    o_log = float((raw[..., :3].double() - ora_raw[..., :3])[ev].abs().max())
    d_map = max(float((out[k].cpu().double() - ora_maps[k]).abs().max()) for k in ora_maps)
    print("ROWS render %s %s %s %s: |gpu - emulation| sigma max %.3e median %.3e logits max %.3e median %.3e; "
          "|gpu - oracle| sigma %.3e logits %.3e maps %.3e; %d of %d rows, stats %s"
          % (name, precision, vdtype, "skip" if skip else "noskip", d_sig, m_sig, d_log, m_log, o_sig, o_log, d_map,
             int(ev.sum()), ev.numel(), stats))
    assert d_sig <= TOL_EMU[("sigma", passes)], d_sig
    assert d_log <= TOL_EMU[("logit", passes)], d_log
    assert m_sig <= TOL_MED[("sigma", passes)] and m_log <= TOL_MED[("logit", passes)], (m_sig, m_log)
    assert o_sig <= GATE_SIGMA[passes] and o_log <= GATE_LOGIT[passes], (o_sig, o_log)
    assert d_map <= GATE_MAP[passes], d_map
