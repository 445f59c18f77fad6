"""GPU: the People-Snapshot mesh path's float64-camera mask test.  nb_mesh_inside_f64 against the reference's own
prepare_inside_pts (tests/golden/mesh_mono_s03.npz) and against its float64 numpy restatement (tools/mesh_mono_case.py) at
full size and on edge cameras; the renderer fed the frame's mask view against the same renderer fed `pts` / `inside`,
bit for bit."""
import numpy as np
import pytest
import torch

from oracle import mesh_case
from tools import mesh_mono_case as MM
from test_mesh_inside_cpu import _module, MESH_RENDERER
from test_mesh_inside_gpu import _grid, _masks, _mesh_renderer, _render, _assert_same_output

pytestmark = pytest.mark.gpu

_cases = {}


@pytest.fixture(scope="module", autouse=True)
def _release_cases():
    yield
    _cases.clear()


def _ren():
    return _module("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)


def _full_case():
    """mono_full: the full-size body, People-Snapshot's 1080 x 1080 camera at ratio 0.5 and a 540 x 540 0 / 255 mask."""
    if "full" not in _cases:
        scene, pkl, _, _ = MM.build_case("mono_full")
        K = MM.get_camera(pkl)["K"].copy()
        K[:2] = K[:2] * MM.RATIO
        msk = MM.silhouette(scene, K, 540, 540, 2)
        _cases["full"] = scene, K, np.eye(3), np.zeros((3, 1)), msk
    return _cases["full"]


def _device_inside(axes, Ks, RTs, msks):
    """grid_inside on numpy inputs (Ks (nv,3,3), RTs (nv,3,4) in their own dtype, msks (nv,H,W)) -> (X,Y,Z) uint8."""
    out = _ren().grid_inside([torch.from_numpy(a).cuda() for a in axes], torch.from_numpy(np.ascontiguousarray(RTs)).cuda(),
                             torch.from_numpy(np.ascontiguousarray(Ks)).cuda(), torch.from_numpy(msks).cuda())
    torch.cuda.synchronize()
    assert out.dtype == torch.uint8 and out.is_cuda
    return out.cpu().numpy()


def _host(axes, Ks, RTs, msks):
    """prepare_inside_pts' float64 projection over the views in order (mesh_case.mesh_inside with a float64 camera); the
    pixel coordinates per view (nv, n, 2) float64 too."""
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inside = mesh_case.mesh_inside(pts, Ks, RTs[:, :, :3], RTs[:, :, 3:], msks)
        p = pts.reshape(-1, 3)
        c = np.stack([(lambda xyz: xyz[:, :2] / xyz[:, 2:])(np.dot(np.dot(p, RT[:, :3].T) + RT[:, 3:].T, K.T))
                      for K, RT in zip(Ks, RTs)])
    return inside, c


def _assert_same_up_to_ties(dev, host, coords, max_frac):
    """dev == host except where some view's numpy coordinate of a differing point lies within 2 float64 ulps of a
    rounding tie k + 0.5 (where the host's BLAS and the kernel's FMA chain may round apart)."""
    diff = np.flatnonzero(dev.reshape(-1) != host.reshape(-1))
    assert len(diff) <= max_frac * dev.size, "%d of %d points differ" % (len(diff), dev.size)
    if len(diff):
        c = coords[:, diff]
        near_tie = np.abs(c - (np.floor(c) + 0.5)) <= 2 * np.spacing(np.abs(c))
        assert near_tie.any(axis=(0, 2)).all(), diff[~near_tie.any(axis=(0, 2))]
    return len(diff)


def _check(axes, Ks, RTs, msks, max_frac=1e-3):
    host, c = _host(axes, Ks, RTs, msks)
    dev = _device_inside(axes, Ks, RTs, msks)
    _assert_same_up_to_ties(dev, host, c, max_frac)
    return dev, host


def test_golden_parity_mesh_mono_s03():
    """The reference's own prepare_inside_pts (golden), bit for bit, from the mask and float64 camera it received; the
    renderer's inside points = pts[inside]."""
    gold = MM.load_golden()
    case = MM.build_case("mono_s03")
    assert MM.case_checksum(*case) == gold["input_sha256"]
    scene = case[0]
    ren = _ren()
    axes = ren.world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    RT = np.concatenate([gold["R"], gold["T"]], axis=1)[None]
    inside = _device_inside(axes, gold["K"][None], RT, gold["msk"][None])
    np.testing.assert_array_equal(inside, gold["inside"])
    assert len(np.unique(inside)) > 2                                          # 0, 255 and values in between
    from neuralbody_b200.lib.config import cfg
    cfg.voxel_size = list(scene["voxel_size"])
    r = ren.Renderer.__new__(ren.Renderer)
    mb = {"wbounds": scene["can_bounds"].cuda(), "RT": torch.from_numpy(RT).cuda(), "Ks": torch.from_numpy(gold["K"][None]).cuda(),
          "msks": torch.from_numpy(gold["msk"][None]).cuda()}
    mb = {k: v[None] if k != "wbounds" else v for k, v in mb.items()}
    wpts, ins = r.grid_from_masks(mb)
    pts = mesh_case.mesh_grid(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    np.testing.assert_array_equal(ins.cpu().numpy(), gold["inside"] != 0)
    want = pts[gold["inside"] != 0]
    assert wpts.shape == (1,) + want.shape
    np.testing.assert_array_equal(wpts[0].cpu().numpy().view(np.int32), want.view(np.int32))


def test_full_size_matches_host():
    scene, K, R, T, msk = _full_case()
    axes = _ren().world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    RT = np.concatenate([R, T], axis=1)[None]
    dev, host = _check(axes, K[None], RT, msk[None], max_frac=1e-5)
    assert 0.05 < (host != 0).mean() < 0.6 and set(np.unique(host)) == {0, 255}
    print("full size: %d of %d points differ (rounding ties)" % (int((dev != host).sum()), dev.size))


def _cameras_f64(nv, H, W, seed, f=None):
    rng = np.random.RandomState(seed)
    from oracle import synth
    Ks, RTs = [], []
    for v in range(nv):
        R, T = synth.look_at_camera(rng.uniform(-0.05, 0.05, 3), 1.6, azimuth_deg=360.0 * v / nv + rng.uniform(0, 10),
                                    elevation_deg=rng.uniform(-20, 20))
        fl = f if f is not None else 0.8 * min(H, W) * rng.uniform(0.9, 1.1)
        Ks.append(np.array([[fl, 0, W / 2.0 + rng.uniform(-3, 3)], [0, fl * rng.uniform(0.95, 1.05), H / 2.0], [0, 0, 1]]))
        RTs.append(np.concatenate([R, T], axis=1))
    return np.stack(Ks).astype(np.float64), np.stack(RTs).astype(np.float64)


@pytest.mark.parametrize("nv", [1, 4])
def test_views_and_mask_values(nv):
    """Masks holding 0, 1 and 255: a point goes on only while it reads exactly 1, inside = the last value read (with one
    view, the mask value itself)."""
    H, W = 64, 64
    dev, host = _check(_grid(), *_cameras_f64(nv, H, W, seed=20 + nv), _masks(nv, H, W, seed=120 + nv, values=(0, 1, 255)))
    assert (host == 1).any() and (host == 0).any() and (host == 255).any()


def test_non_square_mask():
    H, W = 40, 72
    dev, host = _check(_grid(), *_cameras_f64(3, H, W, seed=25), _masks(3, H, W, seed=26))
    assert (host == 1).mean() > 0.01


def test_camera_centre_on_a_grid_point():
    """0 / 0 = NaN for the grid point at the camera centre: astype(int32) gives INT_MIN, the clip 0 -> pixel (0, 0)."""
    H, W = 32, 32
    axes = _grid()
    c = np.array([axes[0][5], axes[1][7], axes[2][11]], np.float64)
    Ks, _ = _cameras_f64(1, H, W, seed=3)
    RT = np.concatenate([np.eye(3), -c.reshape(3, 1)], axis=1)[None]
    for corner in (1, 0):
        msks = np.zeros((1, H, W), np.uint8)
        msks[0, 0, 0] = corner
        msks[0, H // 2:, W // 2:] = 1
        dev, host = _check(axes, Ks, RT, msks)
        assert dev[5, 7, 11] == host[5, 7, 11] == corner


def test_projections_beyond_int32():
    """Pixel coordinates past +-2^31 in float64: astype(int32) gives INT_MIN and the clip 0; coordinates inside the int32
    range but past the image clip to the edge."""
    H, W = 24, 40
    Ks, RTs = _cameras_f64(2, H, W, seed=11, f=1.2e10)
    msks = np.zeros((2, H, W), np.uint8)
    msks[:, :, 0] = 1
    msks[:, 0, :] = 1
    msks[1, :, W - 1] = 2
    axes = _grid()
    dev, host = _check(axes, Ks, RTs, msks)
    _, c = _host(axes, Ks, RTs, msks)
    assert (np.abs(c) > 2.0 ** 31).any() and ((np.abs(c) < 2.0 ** 31) & (np.abs(c) > W)).any()
    assert (host == 1).any() and (host == 0).any()


# ------------------------------------------------------------------------------------------------------------ renderer
def _batches(name):
    """(scene, the grid batch with pts / inside, the mask-view batch) of the golden frame or the full-size one."""
    if name == "mono_s03":
        gold = MM.load_golden()
        scene = MM.build_case("mono_s03")[0]
        K, R, T, msk, inside = gold["K"], gold["R"], gold["T"], gold["msk"], gold["inside"]
    else:
        scene, K, R, T, msk = _full_case()
        axes = _ren().world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
        inside = _device_inside(axes, K[None], np.concatenate([R, T], axis=1)[None], msk[None])   # ties: as the test above
    pts = mesh_case.mesh_grid(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    if name == "mono_full":
        host = MM.mesh_inside_f64(pts, K, R, T, msk)
        assert (host != inside).sum() <= 1e-5 * inside.size
    frame = {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    grid = dict(frame, pts=torch.from_numpy(pts)[None], inside=torch.from_numpy(inside)[None])
    masks = dict(frame, wbounds=scene["can_bounds"], RT=torch.from_numpy(np.concatenate([R, T], axis=1))[None, None],
                 Ks=torch.from_numpy(K)[None, None], msks=torch.from_numpy(msk)[None, None])
    return scene, grid, masks


@pytest.mark.parametrize("name", ["mono_s03", "mono_full"])
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
def test_renderer_mask_batch_equals_grid_batch(name, precision):
    scene, grid, masks = _batches(name)
    assert masks["RT"].dtype == masks["Ks"].dtype == torch.float64
    ren = _mesh_renderer(scene)
    ref = _render(ren, grid, precision)
    out = _render(ren, masks, precision)
    assert len(ref["mesh"].faces) > 1000
    _assert_same_output(out, ref)
    if name == "mono_s03" and precision == "fp32":
        gold = MM.load_golden()
        assert float(np.abs(out["cube"] - gold["cube"]).max()) < 2e-4         # the reference's cube, as test_mesh_gpu holds it
        assert (out["cube"][gold["cube"] == 0] == 0).all()


def test_renderer_rejects_a_mixed_camera():
    scene, _, masks = _batches("mono_s03")
    ren = _mesh_renderer(scene)
    with pytest.raises(ValueError, match="RT and Ks"):
        ren.render({k: v.cuda() for k, v in dict(masks, Ks=masks["Ks"].float()).items()})
    torch.cuda.synchronize()
