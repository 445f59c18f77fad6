"""Distinct-frame case: a B = 3 training batch whose frames differ in everything a frame carries -- pose (Rh / Th and so R),
camera azimuth, feature volumes, latent code and bounds -- so that a kernel reading or writing the wrong frame's slice
changes the result.  Frames 0 and 2 share latent row 2 and are not adjacent; frame 1 uses row 5.  Each frame's bounds
are shifted by b * 0.37 voxel (both rows), which moves the trilinear weights of every sample.
TEST INFRASTRUCTURE ONLY (tests/test_distinct_frames.py, tools/frames_grad_case.py).

The loss reads all five maps: grad_case.loss_of (rgb, depth, acc) + the disp / weights terms of tools/map_grad_case.

Variants: 'middle_empty' moves frame 1's near / far past the far side of the padded ray box, 'all_empty' does that for
every frame, so that none of those samples has a non-zero feature and the training path lists none of them.

The reference is the oracle restatement under autograd in float64 with every float input a leaf (decoder, volumes,
R, Th, bounds, rays, near, far).

The case keeps every sample that carries gradient away from the points where the render is not differentiable: the faces
of the trilinear cells (where d features / d position jumps) and the kinks of the decoder's ReLUs (fc_0..fc_2, view_fc,
and relu(sigma) in raw2outputs).  A float32 kernel computes a sample's position and activations to a few ulps; a sample
within that reach of such a point can land on the other side than the float64 reference, and its position gradient then
differs by O(1).  The per-frame sums of position gradients (R, Th, bounds) cancel heavily, so one such sample moves them
by several 1e-3.  `well_conditioned` redraws the jitter of those samples (and moves a ray that runs along a cell face
sideways by ~0.3 mm), so the gradients compared are functions of the inputs a kernel can be held to."""
import torch

LATENT_INDEX = (2, 5, 2)
BOUNDS_SHIFT_VOXELS = 0.37
N_SAMPLES = 33
N_RAYS = 83
FACE_MARGIN = 2e-4      # cells (float32 rounding of a position is ~1e-5 cell at level 0)
RELU_MARGIN = 3e-5      # of the rms pre-activation of that layer (float32 / TF32x3 GEMM rounding: ~1e-6)
VARIANTS = ("distinct", "middle_empty", "all_empty")
# (Rh, Th, camera azimuth, volume seed) per frame
POSES = (((0.30, -0.20, 0.10), (0.10, 0.20, 1.00), 20.0, 313),
         ((0.22, -0.05, 0.25), (0.16, 0.17, 1.03), 105.0, 318),
         ((0.36, -0.32, 0.02), (0.04, 0.24, 0.96), 230.0, 323))
FRAME_KEYS = ("coord", "out_sh", "bounds", "can_bounds", "R", "Th", "latent_index", "ray_o", "ray_d", "near", "far")
# inputs with a leading frame axis whose gradient the tests compare per frame
FRAME_GRADS = ("R", "Th", "bounds", "ray_o", "ray_d", "near", "far", "vol0", "vol1", "vol2", "vol3")
LEAVES = ("R", "Th", "bounds", "ray_o", "ray_d", "near", "far")


def _ray_subset(total, n, W):
    """n rays spread over the image (row-major pixels); one ray: the centre pixel, which sees the body."""
    if n == 1:
        return torch.tensor([(total // W // 2) * W + W // 2])
    return (torch.arange(n) * total) // n + (total // n) // 2


def build(n_samples=N_SAMPLES, n_rays=N_RAYS, variant="distinct", batch=3, frames=None, volume_dtype=None, subnormal=False):
    """(scene, t_rand, G, Gm): `batch` frames (or the frames listed in `frames`) of the distinct case, n_rays rays each,
    jitter t_rand (B,n,S) and the cotangents G (rgb, depth, acc; grad_case.loss_of) and Gm (disp, weights;
    map_grad_case.loss_of), all from seed 77 -- drawn for the full 3-frame batch and sliced, so a sub-batch sees the same
    numbers as those frames of the full one.
    volume_dtype (e.g. torch.float16): every volume is rounded to it (synth.round_volumes; `subnormal` scales level 0 into
    the fp16 subnormal range first) BEFORE the samples are conditioned, since the rounding moves the decoder's
    pre-activations and the kink margins must hold on the volumes the kernels read."""
    from oracle import synth
    assert variant in VARIANTS, variant
    ids = list(range(batch)) if frames is None else list(frames)
    parts = []
    for b in range(max(3, max(ids) + 1)):
        Rh, Th, az, vs = POSES[b % 3]
        f = synth.make_scene(H=24, W=24, scale=0.25, all_hit=True, latent_index=LATENT_INDEX[b % 3], Rh=Rh, Th=Th,
                             azimuth_deg=az, volume_seed=vs)
        idx = _ray_subset(f["ray_o"].shape[1], n_rays, 24)
        for k in ("ray_o", "ray_d", "near", "far"):
            f[k] = f[k][:, idx].contiguous()
        shift = b * BOUNDS_SHIFT_VOXELS * torch.tensor(f["voxel_size"], dtype=torch.float32)
        f["bounds"] = (f["bounds"] + shift).contiguous()
        parts.append(f)
    assert all(torch.equal(p["out_sh"], parts[0]["out_sh"]) for p in parts), "frames must share out_sh (one volume shape)"
    full = len(parts)
    n = parts[0]["ray_o"].shape[1]
    scene = {k: torch.cat([p[k] for p in parts], 0).contiguous() for k in FRAME_KEYS}
    scene["volumes"] = [torch.cat([p["volumes"][l] for p in parts], 0).contiguous() for l in range(4)]
    scene["weights"], scene["voxel_size"] = parts[0]["weights"], parts[0]["voxel_size"]
    if volume_dtype is not None:
        scene["volumes"] = synth.round_volumes(scene["volumes"], volume_dtype, subnormal)
    else:
        assert not subnormal, "the subnormal variant is a rounded case (volume_dtype)"
    empty = {"distinct": (), "middle_empty": (1,), "all_empty": tuple(range(3))}[variant]
    for b in empty:
        # beyond the far side of the padded box the ray only moves away from the body: every sample has zero features
        far = scene["far"][b].clone()
        scene["near"][b], scene["far"][b] = far + 0.10, far + 0.30
    g = torch.Generator().manual_seed(77)
    t_rand = torch.rand((full, n, n_samples), generator=g)
    G = {"rgb_map": torch.randn((full, n, 3), generator=g), "depth_map": torch.randn((full, n), generator=g) * 0.3,
         "acc_map": torch.randn((full, n), generator=g) * 0.5}
    Gm = (torch.randn((full, n), generator=g) * 0.2, torch.randn((full, n, n_samples), generator=g) * 0.5)
    t_rand = well_conditioned(scene, t_rand, g)
    sel = torch.tensor(ids)
    for k in FRAME_KEYS:
        scene[k] = scene[k][sel].contiguous()
    scene["volumes"] = [v[sel].contiguous() for v in scene["volumes"]]
    return scene, t_rand[sel].contiguous(), {k: v[sel].contiguous() for k, v in G.items()}, tuple(t[sel].contiguous() for t in Gm)


def fragile_samples(scene, t_rand):
    """(B,n,S) bool, in float64: the samples with a non-zero feature that lie within FACE_MARGIN cells of a trilinear cell
    face of any level (grid_sample align_corners=True index space), or have a ReLU pre-activation within RELU_MARGIN of
    zero.  A sample with all-zero features has sigma(empty) < 0 and weight 0: no gradient flows through it."""
    from oracle import neuralbody_oracle as O
    sc = to_double(scene)
    _, z_vals = O.get_sampling_points(sc["ray_o"], sc["ray_d"], sc["near"], sc["far"], t_rand.shape[2], 1.0, True,
                                      t_rand.double())
    return sample_conditions(scene, z_vals)["fragile"]


def sample_conditions(scene, z_vals, scale=None, kinks=True):
    """What fragile_samples decides, for the samples at the depths z_vals (B,n,S) along the scene's rays, in float64.
    Returns dict of (B,n,S) tensors: 'fragile', 'occupied' (a non-zero feature), 'face' (distance in cells to the nearest
    trilinear cell face of any level), and 'scale': the rms pre-activation of each ReLU layer over the occupied samples, the
    unit of RELU_MARGIN.  `scale` given: judge against those rms values instead, so that a subset of samples (redrawn ones)
    is held to the margins of the whole set it belongs to.  kinks=False: 'occupied' and 'face' only (no decoder run)."""
    from oracle import neuralbody_oracle as O
    sc = to_double(scene)
    B, n, S = z_vals.shape
    pts = sc["ray_o"][:, :, None] + sc["ray_d"][:, :, None] * z_vals.double()[..., None]   # get_sampling_points' pts
    pts = pts.reshape(B, n * S, 3)
    sp = O.prepare_sp_input(sc)
    grid = O.get_grid_coords(O.pts_to_can_pts(pts, sp["R"], sp["Th"]), sp["bounds"], sp["out_sh"], sc["voxel_size"])
    face = torch.full((B, n * S), float("inf"), dtype=torch.float64)
    for v in sc["volumes"]:
        size = torch.tensor([v.shape[4], v.shape[3], v.shape[2]], dtype=torch.float64)   # x, y, z = W, H, D
        idx = (grid + 1) / 2 * (size - 1)
        face = torch.minimum(face, (idx - idx.round()).abs().min(-1).values)
    w = sc["weights"]
    feats = O.interpolate_features(grid, sc["volumes"])                               # (B, 352, P)
    occupied = (feats != 0).any(1)
    if not kinks:
        return {"occupied": occupied.view(B, n, S), "face": face.view(B, n, S)}
    pre = []
    h = feats
    for name in ("fc_0", "fc_1", "fc_2"):
        z = O._conv(w, name, h)
        pre.append(z)
        h = torch.relu(z)
    pre.append(O._conv(w, "alpha_fc", h))
    lat = w["latent.weight"][sc["latent_index"]][..., None].expand(B, 128, n * S)
    f = O._conv(w, "latent_fc", torch.cat((O._conv(w, "feature_fc", h), lat), 1))
    viewdir = (sc["ray_d"] / torch.norm(sc["ray_d"], dim=2, keepdim=True))[:, :, None].expand(B, n, S, 3).reshape(B, n * S, 3)
    f = torch.cat((f, O.positional_embed(viewdir, 4).transpose(1, 2), O.positional_embed(pts, 10).transpose(1, 2)), 1)
    pre.append(O._conv(w, "view_fc", f))
    kink = torch.zeros((B, n * S), dtype=torch.bool)
    rms_of = []
    for i, z in enumerate(pre):
        live = occupied[:, None].expand_as(z)
        rms = float(z[live].pow(2).mean().sqrt()) if bool(live.any()) else 1.0
        rms = rms if scale is None else scale[i]
        rms_of.append(rms)
        kink |= (z.abs() < RELU_MARGIN * rms).any(1)
    return {"fragile": (occupied & ((face < FACE_MARGIN) | kink)).view(B, n, S), "occupied": occupied.view(B, n, S),
            "face": face.view(B, n, S), "scale": rms_of}


def well_conditioned(scene, t_rand, gen):
    """t_rand with the draws of fragile_samples redrawn from `gen` until none is left; a ray with a sample that is fragile
    again after its redraw runs along a cell face and is moved sideways by ~0.3 mm (scene['ray_o'], in place)."""
    t_rand = t_rand.clone()
    prev = None
    for it in range(40):
        bad = fragile_samples(scene, t_rand)
        if not bool(bad.any()):
            return t_rand
        t_rand[bad] = torch.rand(int(bad.sum()), generator=gen)
        if prev is not None:
            rays = (bad & prev).any(-1)          # fragile again after a redraw: the ray runs along a cell face
            scene["ray_o"][rays] += 3e-4 * torch.randn((int(rays.sum()), 3), generator=gen)
        prev = bad
    raise AssertionError("could not keep the samples off the cell faces and ReLU kinks")


def loss_of(ret, G, Gm):
    from tools import map_grad_case as MC
    return MC.loss_of(ret, G, Gm)


def to_double(scene):
    sc = dict(scene)
    for k in LEAVES + ("can_bounds",):
        sc[k] = scene[k].double()
    sc["weights"] = {k: v.double() for k, v in scene["weights"].items()}
    sc["volumes"] = [v.double() for v in scene["volumes"]]
    return sc


def leaves(scene):
    """A copy of the scene whose float inputs are all fresh leaves requiring grad."""
    sc = dict(scene)
    for k in LEAVES:
        sc[k] = scene[k].clone().requires_grad_(True)
    sc["weights"] = {k: v.clone().requires_grad_(True) for k, v in scene["weights"].items()}
    sc["volumes"] = [v.clone().requires_grad_(True) for v in scene["volumes"]]
    return sc


def grads_of(sc):
    from oracle import grad_case
    out = {k: sc[k].grad for k in LEAVES}
    out.update({k: sc["weights"][k].grad for k in grad_case.GRAD_KEYS})
    out.update({"vol%d" % l: v.grad for l, v in enumerate(sc["volumes"])})
    return out


def oracle_grads(scene, t_rand, G, Gm, n_samples, dtype=torch.float64):
    """Autograd of loss_of through the oracle restatement in `dtype`, every float input a leaf -> ({name: grad}, outputs)."""
    from oracle import neuralbody_oracle as O
    sc = leaves(to_double(scene) if dtype == torch.float64 else scene)
    ret = O.render(sc, n_samples=n_samples, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand.to(dtype))
    loss_of(ret, {k: v.to(dtype) for k, v in G.items()}, tuple(t.to(dtype) for t in Gm)).backward()
    return grads_of(sc), {k: v.detach() for k, v in ret.items()}
