"""GPU: the mesh renderer's mask-view path.  nb_mesh_inside against the reference's own prepare_inside_pts
(tests/golden/mesh_s03.npz) and against its numpy restatement (oracle/mesh_case.mesh_inside) at full size and on edge
cameras; the renderer fed the frame's mask views against the same renderer fed `pts` / `inside`, bit for bit."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import mesh_case, synth
import gpu_utils as G
from test_mesh_inside_cpu import dataset_item

pytestmark = pytest.mark.gpu

MESH_RENDERER = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")

_cases = {}


@pytest.fixture(scope="module", autouse=True)
def _release_cases():
    """The cases (the full-size one holds the 97 MB grid and the volumes) live for this module only."""
    yield
    _cases.clear()


def _case(name):
    if name not in _cases:
        _cases[name] = mesh_case.build_case(name)
    return _cases[name]


def _ren_module():
    from neuralbody_b200.lib.networks.make_network import load_source
    return load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)


def _device_inside(axes, Ks, Rs, Ts, msks):
    """nb_mesh_inside on numpy inputs (Ks (nv,3,3), Rs (nv,3,3), Ts (nv,3,1), msks (nv,H,W)) -> (X,Y,Z) uint8."""
    RT = np.concatenate([Rs, Ts], axis=2).astype(np.float32)
    out = _ren_module().grid_inside([torch.from_numpy(a).cuda() for a in axes], torch.from_numpy(RT).cuda(),
                                    torch.from_numpy(np.asarray(Ks, np.float32)).cuda(), torch.from_numpy(msks).cuda())
    torch.cuda.synchronize()
    assert out.dtype == torch.uint8 and out.is_cuda
    return out.cpu().numpy()


def _host_coords(pts, Ks, Rs, Ts):
    """base_utils.project as prepare_inside_pts calls it, per view: (nv, n, 2) float32."""
    out = []
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for v in range(len(Ks)):
            RT = np.concatenate([Rs[v], Ts[v]], axis=1)
            xyz = np.dot(pts, RT[:, :3].T) + RT[:, 3:].T
            xyz = np.dot(xyz, Ks[v].T)
            out.append(xyz[:, :2] / xyz[:, 2:])
    return np.stack(out)


def _assert_same_up_to_ties(dev, host, axes, Ks, Rs, Ts, max_frac=1e-5):
    """dev == host except where the host's BLAS and the kernel's FMA chain may round a pixel coordinate to different sides
    of a rounding tie: for every differing point, some view's numpy coordinate lies within 2 float32 ulps of k + 0.5."""
    assert dev.shape == host.shape
    diff = np.argwhere(dev != host)
    assert len(diff) <= max_frac * dev.size, "%d of %d points differ" % (len(diff), dev.size)
    if len(diff):
        pts = np.stack([axes[0][diff[:, 0]], axes[1][diff[:, 1]], axes[2][diff[:, 2]]], axis=1)
        c = _host_coords(pts, Ks, Rs, Ts)                                   # (nv, d, 2)
        near_tie = np.abs(c - (np.floor(c) + 0.5)) <= 2 * np.spacing(np.abs(c).astype(np.float32))
        assert near_tie.any(axis=(0, 2)).all(), diff[~near_tie.any(axis=(0, 2))]
    return len(diff)


def test_golden_parity_mesh_s03():
    """The reference's own prepare_inside_pts (golden), bit for bit; the inside points = pts[inside]."""
    gold = mesh_case.load_golden()
    scene, masks, batch = _case("mesh_s03")
    assert mesh_case.case_checksum(scene, masks) == gold["input_sha256"]
    ren = _ren_module()
    axes = ren.world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    inside = _device_inside(axes, *mesh_case._views(masks))
    np.testing.assert_array_equal(inside, gold["inside"])
    # the renderer's inside points against upstream's boolean indexing of the grid
    from neuralbody_b200.lib.config import cfg
    cfg.voxel_size = list(scene["voxel_size"])
    r = ren.Renderer.__new__(ren.Renderer)
    mb = {"wbounds": scene["can_bounds"].cuda(), "RT": masks["RT"].cuda(), "Ks": masks["Ks"].cuda(), "msks": masks["msks"].cuda()}
    wpts, ins = r.grid_from_masks(mb)
    pts = mesh_case.mesh_grid(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    np.testing.assert_array_equal(ins.cpu().numpy(), gold["inside"].astype(bool))
    want = pts[gold["inside"] == 1]
    assert wpts.shape == (1,) + want.shape
    np.testing.assert_array_equal(wpts[0].cpu().numpy().view(np.int32), want.view(np.int32))


def test_full_size_matches_host():
    """mesh_full: 170 x 325 x 146 = 8.07 M points, 4 views, against mesh_case.mesh_inside computed here."""
    scene, masks, batch = _case("mesh_full")
    axes = _ren_module().world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    views = mesh_case._views(masks)
    dev = _device_inside(axes, *views)
    host = batch["inside"][0].numpy()
    assert dev.shape == (170, 325, 146) and 0.05 < host.mean() < 0.5
    n = _assert_same_up_to_ties(dev, host, axes, *views[:3])
    print("full size: %d of %d points differ (rounding ties)" % (n, dev.size))


# ------------------------------------------------------------------------------------------------------------ renderer
def _mesh_renderer(scene):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer
    net, _ = G.make_net_and_renderer(scene)
    old = cfg.renderer_module, cfg.renderer_path
    cfg.renderer_module, cfg.renderer_path = "neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER
    try:
        ren = make_renderer(cfg, net)
    finally:
        cfg.renderer_module, cfg.renderer_path = old
    return ren


def _render(ren, batch, precision, mesh_th=10.0):
    from neuralbody_b200.lib.config import cfg
    old = {k: cfg[k] for k in ("mesh_th", "density_precision") if k in cfg}
    cfg.mesh_th, cfg.density_precision = mesh_th, precision
    try:
        with torch.no_grad():
            out = ren.render({k: v.cuda() for k, v in batch.items()})
    finally:
        cfg.pop("density_precision", None)
        cfg.update(old)
    return out


def _mask_batch(batch, scene, masks):
    b = {k: v for k, v in batch.items() if k not in ("pts", "inside")}
    b.update(wbounds=scene["can_bounds"], RT=masks["RT"], Ks=masks["Ks"], msks=masks["msks"])
    return b


def _assert_same_output(a, b):
    assert a["cube"].shape == b["cube"].shape and np.array_equal(a["cube"].view(np.int64), b["cube"].view(np.int64))
    np.testing.assert_array_equal(np.asarray(a["mesh"].vertices).view(np.int64), np.asarray(b["mesh"].vertices).view(np.int64))
    np.testing.assert_array_equal(np.asarray(a["mesh"].faces), np.asarray(b["mesh"].faces))


@pytest.mark.parametrize("name", ["mesh_s03", "mesh_full"])
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
def test_renderer_mask_batch_equals_grid_batch(name, precision):
    scene, masks, batch = _case(name)
    ren = _mesh_renderer(scene)
    ref = _render(ren, batch, precision)
    mb = _mask_batch(batch, scene, masks)
    out = _render(ren, mb, precision)
    if name == "mesh_full":
        # the grid batch's inside is the host's; a rounding tie (test_full_size_matches_host) would move a point
        dev = _device_inside(_ren_module().world_axes(scene["can_bounds"][0].numpy(), scene["voxel_size"]),
                             *mesh_case._views(masks))
        if not np.array_equal(dev, batch["inside"][0].numpy()):
            batch = dict(batch, inside=torch.from_numpy(dev)[None])
            ref = _render(ren, batch, precision)
    assert len(ref["mesh"].faces) > 1000
    _assert_same_output(out, ref)
    _assert_same_output(_render(ren, mb, precision), out)                   # two runs, identical


def test_renderer_with_the_dataset_drop_in():
    """The drop-in's item, collated as the reference's DataLoader does, renders the golden frame's cube."""
    from torch.utils.data import default_collate
    scene, masks, batch = _case("mesh_s03")
    item = default_collate([dataset_item(scene, masks)])
    assert "pts" not in item and "inside" not in item
    ren = _mesh_renderer(scene)
    _assert_same_output(_render(ren, item, "fp32", 15.0), _render(ren, batch, "fp32", 15.0))


# ------------------------------------------------------------------------------------------------------------ edges
def _grid(n=(17, 19, 23), lo=(-0.4, -0.5, -0.3), hi=(0.4, 0.5, 0.3)):
    return [np.linspace(lo[a], hi[a], n[a]).astype(np.float32) + np.float32(0.0013 * (a + 1)) for a in range(3)]


def _cameras(nv, H, W, seed, distance=1.6, f=None):
    rng = np.random.RandomState(seed)
    Ks, Rs, Ts = [], [], []
    for v in range(nv):
        R, T = synth.look_at_camera(rng.uniform(-0.05, 0.05, 3), distance, azimuth_deg=360.0 * v / nv + rng.uniform(0, 10),
                                    elevation_deg=rng.uniform(-20, 20))
        fl = f if f is not None else 0.8 * min(H, W) * rng.uniform(0.9, 1.1)
        Ks.append(np.array([[fl, 0, W / 2.0 + rng.uniform(-3, 3)], [0, fl * rng.uniform(0.95, 1.05), H / 2.0], [0, 0, 1]]))
        Rs.append(R); Ts.append(T)
    return tuple(np.stack(x).astype(np.float32) for x in (Ks, Rs, Ts))


def _masks(nv, H, W, seed, values=(0, 1)):
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[:H, :W]
    m = []
    for v in range(nv):
        cy, cx, r = H * rng.uniform(0.3, 0.7), W * rng.uniform(0.3, 0.7), min(H, W) * rng.uniform(0.2, 0.4)
        blob = ((yy - cy) ** 2 + (xx - cx) ** 2 < r * r).astype(np.uint8)
        noise = rng.choice(values, size=(H, W)).astype(np.uint8)
        m.append(np.where(rng.rand(H, W) < 0.1, noise, blob))
    return np.stack(m).astype(np.uint8)


def _check(axes, Ks, Rs, Ts, msks):
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        host = mesh_case.mesh_inside(pts, Ks, Rs, Ts, msks)
    dev = _device_inside(axes, Ks, Rs, Ts, msks)
    _assert_same_up_to_ties(dev, host, axes, Ks, Rs, Ts, max_frac=1e-3)
    return dev, host


@pytest.mark.parametrize("nv", [1, 4, 21])
def test_views_in_order_and_mask_values(nv):
    """nv = 1 / 4 / 21 views; masks holding 0, 1 and 2: a point goes on only while it reads exactly 1, and inside is the
    last value read (2 stops the loop and stays 2)."""
    H, W = 64, 64
    axes = _grid()
    dev, host = _check(axes, *_cameras(nv, H, W, seed=nv), _masks(nv, H, W, seed=100 + nv, values=(0, 1, 2)))
    assert (host == 1).any() and (host == 0).any() and (host == 2).any()


def test_non_square_mask():
    H, W = 40, 72
    dev, host = _check(_grid(), *_cameras(3, H, W, seed=5), _masks(3, H, W, seed=6))
    assert (host == 1).mean() > 0.01


def test_camera_seeing_the_grid_from_behind():
    """A camera inside the grid: the points behind it (z < 0) project through the centre, mirrored, as numpy projects them."""
    H, W = 48, 56
    Ks, Rs, Ts = _cameras(2, H, W, seed=9)
    Rs[1] = np.eye(3, dtype=np.float32)
    Ts[1] = np.array([[0.013], [-0.021], [0.017]], np.float32)             # centre at (-0.013, 0.021, -0.017), inside the box
    axes = _grid()
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1).reshape(-1, 3)
    assert (pts[:, 2] + Ts[1, 2, 0] < 0).mean() > 0.3                         # a third of the grid is behind the camera
    msks = np.ones((2, H, W), np.uint8)
    msks[1] = _masks(1, H, W, seed=10)[0]
    dev, host = _check(axes, Ks, Rs, Ts, msks)
    assert (host == 0).any() and (host == 1).any()


def test_camera_centre_on_a_grid_point():
    """0 / 0 = NaN for the grid point at the camera centre: astype(int32) gives INT_MIN, the clip 0, so it reads pixel
    (0, 0) -- inside where that pixel is 1 whatever its neighbours."""
    H, W = 32, 32
    axes = _grid()
    c = np.array([axes[0][5], axes[1][7], axes[2][11]], np.float32)
    Ks, _, _ = _cameras(1, H, W, seed=3)
    Rs = np.eye(3, dtype=np.float32)[None]
    Ts = (-c).reshape(1, 3, 1)
    for corner in (1, 0):
        msks = np.zeros((1, H, W), np.uint8)
        msks[0, 0, 0] = corner
        msks[0, H // 2:, W // 2:] = 1
        dev, host = _check(axes, Ks, Rs, Ts, msks)
        assert dev[5, 7, 11] == host[5, 7, 11] == corner


def test_projections_beyond_int32():
    """Pixel coordinates past +-2^31: astype(int32) gives INT_MIN and the clip 0 (pixel 0, not W - 1); coordinates inside the
    int32 range but past the image clip to the edge."""
    H, W = 24, 40
    Ks, Rs, Ts = _cameras(2, H, W, seed=11, f=1.2e10)
    msks = np.zeros((2, H, W), np.uint8)
    msks[:, :, 0] = 1                                  # column 0 in, column W - 1 out
    msks[:, 0, :] = 1                                  # row 0 in, row H - 1 out
    msks[1, :, W - 1] = 2
    axes = _grid()
    dev, host = _check(axes, Ks, Rs, Ts, msks)
    pts = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1).reshape(-1, 3)
    c = _host_coords(pts, Ks, Rs, Ts)
    assert (np.abs(c) > 2.0 ** 31).any() and ((np.abs(c) < 2.0 ** 31) & (np.abs(c) > W)).any()
    assert (host == 1).any() and (host == 0).any()


# ------------------------------------------------------------------------------------------------------------ rejections
def test_rejections():
    scene, masks, batch = _case("mesh_s03")
    ren = _mesh_renderer(scene)
    mb = {k: v.cuda() for k, v in _mask_batch(batch, scene, masks).items()}
    for k in ("wbounds", "RT", "Ks", "msks"):
        with pytest.raises(KeyError, match=r"pts.*inside.*wbounds.*RT.*Ks.*msks"):
            ren.render({kk: v for kk, v in mb.items() if kk != k})
    with pytest.raises(ValueError, match="msks"):                               # mask views of different counts
        ren.render(dict(mb, RT=mb["RT"][:, :3]))
    with pytest.raises(ValueError, match="msks"):
        ren.render(dict(mb, Ks=mb["Ks"][:, :, :2]))
    with pytest.raises(ValueError, match="msks"):
        ren.render(dict(mb, msks=mb["msks"][0]))
    with pytest.raises(ValueError, match="nv >= 1"):                            # nv = 0
        ren.render(dict(mb, msks=mb["msks"][:, :0], RT=mb["RT"][:, :0], Ks=mb["Ks"][:, :0]))
    for k in ("RT", "Ks", "msks"):
        with pytest.raises(RuntimeError, match="CUDA"):
            ren.render(dict(mb, **{k: mb[k].cpu()}))
    ri = _ren_module()
    axes = [torch.zeros(3, device="cuda")] * 3
    with pytest.raises(RuntimeError, match="CUDA"):
        ri.grid_inside([a.cpu() for a in axes], mb["RT"][0], mb["Ks"][0], mb["msks"][0])
    with pytest.raises(ValueError, match="nv"):
        ri.grid_inside(axes, mb["RT"][0, :2], mb["Ks"][0], mb["msks"][0])
    torch.cuda.synchronize()
