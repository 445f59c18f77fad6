"""The mesh renderer's inputs and golden vectors (TEST INFRASTRUCTURE ONLY).

`mesh_grid` / `mesh_inside` restate the mesh dataset's world grid and its mask-view test
(lib/datasets/light_stage/multi_view_mesh_dataset.py:121-160) with the synthetic silhouettes of `synth.make_mask_views`
standing in for the dataset's CIHP masks.  `build_case` assembles a mesh-renderer batch from them.

    python -m oracle.mesh_case

(in the build container, where the reference tree exists) writes tests/golden/mesh_s03.npz by running the UNMODIFIED
reference: the grid and `inside` come from its own `Dataset.__getitem__` / `prepare_inside_pts` (called unbound on a
stand-in `self` whose `get_mask` returns the synthetic mask), and the cube from its own
`if_mesh_renderer.Renderer.render`, with `mcubes` / `trimesh` replaced by stubs (the `mcubes` stub records the cube it
is handed)."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh_s03.npz")

# name -> (scene kwargs, mask-view kwargs)
CASES = {
    # scale-0.3 body: a 52 x 99 x 59 grid (304 k points), cheap on the CPU
    "mesh_s03": (dict(H=16, W=16, scale=0.3, all_hit=True), dict(nv=4, H=96, W=96, radius=2)),
    # the full-size synth-313 body on its 5 mm grid (170 x 325 x 146 = 8.07 M points)
    "mesh_full": (dict(H=16, W=16, scale=1.0, all_hit=True), dict(nv=4, H=256, W=256, radius=3)),
}


def mesh_grid(can_bounds, voxel_size):
    """multi_view_mesh_dataset.py:150-160: the world grid (X,Y,Z,3) float32 over can_bounds (2,3) float32."""
    x = np.arange(can_bounds[0, 0], can_bounds[1, 0] + voxel_size[0], voxel_size[0])
    y = np.arange(can_bounds[0, 1], can_bounds[1, 1] + voxel_size[1], voxel_size[1])
    z = np.arange(can_bounds[0, 2], can_bounds[1, 2] + voxel_size[2], voxel_size[2])
    pts = np.stack(np.meshgrid(x, y, z, indexing='ij'), axis=-1)
    return pts.astype(np.float32)


def mesh_inside(pts, Ks, Rs, Ts, msks):
    """multi_view_mesh_dataset.py:121-148 (prepare_inside_pts with base_utils.project): 1 where a grid point projects into
    the foreground of every view, views taken in order on the points still inside.  Ks (nv,3,3), Rs (nv,3,3),
    Ts (nv,3,1) world->camera in metres, msks (nv,H,W) uint8."""
    sh = pts.shape
    pts3d = pts.reshape(-1, 3)
    inside = np.ones([len(pts3d)]).astype(np.uint8)
    for nv in range(len(msks)):
        ind = inside == 1
        pts3d_ = pts3d[ind]
        RT = np.concatenate([Rs[nv], Ts[nv]], axis=1)
        xyz = np.dot(pts3d_, RT[:, :3].T) + RT[:, 3:].T
        xyz = np.dot(xyz, Ks[nv].T)
        pts2d = xyz[:, :2] / xyz[:, 2:]
        msk = msks[nv]
        H, W = msk.shape
        pts2d = np.round(pts2d).astype(np.int32)
        pts2d[:, 0] = np.clip(pts2d[:, 0], 0, W - 1)
        pts2d[:, 1] = np.clip(pts2d[:, 1], 0, H - 1)
        inside[ind] = msk[pts2d[:, 1], pts2d[:, 0]]
    return inside.reshape(*sh[:-1])


def _views(masks):
    RT = masks["RT"][0].numpy()
    return masks["Ks"][0].numpy(), RT[:, :, :3], RT[:, :, 3:], masks["msks"][0].numpy()


def build_case(name):
    """-> (scene, masks, batch) with batch = the mesh dataset's item as default_collate hands it to the renderer
    (CPU tensors): coord / out_sh / bounds / R / Th / latent_index of the scene, pts (1,X,Y,Z,3), inside (1,X,Y,Z)."""
    from oracle import synth
    skw, mkw = CASES[name]
    scene = synth.make_scene(**skw)
    masks = synth.make_mask_views(scene, **mkw)
    pts = mesh_grid(scene["can_bounds"][0].numpy(), scene["voxel_size"])
    inside = mesh_inside(pts, *_views(masks))
    batch = {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    batch["pts"] = torch.from_numpy(pts)[None]
    batch["inside"] = torch.from_numpy(inside)[None]
    return scene, masks, batch


def case_checksum(scene, masks):
    """sha256 over everything the mesh render consumes (grid inputs, mask views, volumes, weights)."""
    h = hashlib.sha256()
    for k in ("coord", "out_sh", "bounds", "can_bounds", "R", "Th", "latent_index"):
        h.update(scene[k].contiguous().numpy().tobytes())
    for k in ("RT", "Ks", "msks"):
        h.update(masks[k].contiguous().numpy().tobytes())
    for v in scene["volumes"]:
        h.update(v.contiguous().numpy().tobytes())
    for k in sorted(scene["weights"]):
        h.update(scene["weights"][k].contiguous().numpy().tobytes())
    return h.hexdigest()


def load_golden(path=GOLDEN):
    """-> dict: shape (X,Y,Z), inside (X,Y,Z) uint8, sigma (n_inside,) float32, pts_sha256, input_sha256, cube (padded
    float64, rebuilt as upstream builds it)."""
    from oracle import mcubes_oracle
    z = np.load(path)
    shape = tuple(int(s) for s in z["shape"])
    inside = np.unpackbits(z["inside_bits"])[:int(np.prod(shape))].reshape(shape)
    out = {"shape": shape, "inside": inside, "sigma": z["sigma"], "pts_sha256": bytes(z["pts_sha256"]).decode(),
           "input_sha256": bytes(z["input_sha256"]).decode()}
    out["cube"] = mcubes_oracle.pad_cube(inside, out["sigma"].astype(np.float64))
    return out


# ----------------------------------------------------------------------------- generator (needs the reference tree)
def _reference_item(scene, masks):
    """The reference's Dataset.__getitem__(0) on a stand-in `self`: vertices / params written to a temp dir (as
    make_golden.data_golden does), get_mask -> the synthetic silhouettes."""
    import tempfile
    import types
    from oracle import ref_harness, synth
    cfg = ref_harness.load_reference()[0]
    for name in ("trimesh", "imageio", "plyfile"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.PlyData = object
            sys.modules[name] = m
    from lib.datasets.light_stage import multi_view_mesh_dataset as ref_mds
    Ks, Rs, Ts, msks = _views(masks)
    Rh, Th = np.array([0.3, -0.2, 0.1]), np.array([[0.1, 0.2, 1.0]])      # synth.make_scene's defaults
    world = scene["verts_world"].numpy()
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "vertices")); os.makedirs(os.path.join(d, "params"))
        np.save(os.path.join(d, "vertices", "0.npy"), world)
        np.save(os.path.join(d, "params", "0.npy"), {"Rh": Rh.reshape(1, 3), "Th": Th})
        cfg.vertices, cfg.params, cfg.big_box = "vertices", "params", False
        cfg.voxel_size = [float(v) for v in scene["voxel_size"]]
        cfg.begin_ith_frame, cfg.num_train_frame = 0, int(scene["weights"]["latent.weight"].shape[0])
        fake = types.SimpleNamespace(data_root=d, human="synth", ims=np.zeros((1, len(msks))), Ks=Ks, Rs=Rs, Ts=Ts,
                                     get_mask=lambda i, nv: msks[nv])
        fake.prepare_input = lambda i: ref_mds.Dataset.prepare_input(fake, i)
        fake.prepare_inside_pts = lambda pts, i: ref_mds.Dataset.prepare_inside_pts(fake, pts, i)
        item = ref_mds.Dataset.__getitem__(fake, 0)
    assert np.array_equal(item["out_sh"], scene["out_sh"][0].numpy()) and np.array_equal(item["coord"], scene["coord"][0].numpy())
    assert np.array_equal(item["wbounds"], scene["can_bounds"][0].numpy())
    assert np.allclose(synth._rodrigues(Rh), item["R"], atol=1e-6)
    return item


def _reference_cube(scene, batch):
    """The reference's if_mesh_renderer.Renderer.render with mcubes / trimesh stubbed; returns ret['cube']."""
    import types
    from oracle import ref_harness
    cfg, latent_xyzc, _, _ = ref_harness.load_reference()
    seen = {}

    def marching_cubes(cube, th):
        seen["cube"], seen["th"] = cube.copy(), th
        return np.zeros((0, 3)), np.zeros((0, 3), np.int64)

    mc = types.ModuleType("mcubes")
    mc.marching_cubes = marching_cubes
    tm = types.ModuleType("trimesh")
    tm.Trimesh = lambda v, f: ("mesh", v, f)
    old = {k: sys.modules.get(k) for k in ("mcubes", "trimesh")}
    sys.modules["mcubes"], sys.modules["trimesh"] = mc, tm
    try:
        from lib.networks.renderer import if_mesh_renderer
        cfg.voxel_size = [float(v) for v in scene["voxel_size"]]
        cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
        net = latent_xyzc.Network()
        missing, unexpected = net.load_state_dict(scene["weights"], strict=False)
        assert not unexpected and all(k.startswith("xyzc_net") or k.startswith("c.") for k in missing)
        net.eval()
        net.encode_sparse_voxels = lambda sp_input: scene["volumes"]
        with torch.no_grad():
            ret = if_mesh_renderer.Renderer(net).render(batch)
    finally:
        for k, v in old.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    assert np.array_equal(ret["cube"], seen["cube"]) and seen["th"] == cfg.mesh_th
    return ret["cube"]


def make_golden(name="mesh_s03"):
    scene, masks, batch = build_case(name)
    item = _reference_item(scene, masks)
    pts, inside = item["pts"], item["inside"]
    batch = dict(batch)
    batch["pts"], batch["inside"] = torch.from_numpy(pts)[None], torch.from_numpy(inside)[None]
    cube = _reference_cube(scene, batch)
    assert cube.dtype == np.float64 and cube.shape == tuple(s + 20 for s in inside.shape)
    core = cube[10:-10, 10:-10, 10:-10]
    sigma = core[inside == 1].astype(np.float32)
    assert np.array_equal(sigma.astype(np.float64), core[inside == 1])     # float32 values held in float64
    arrays = {"shape": np.array(inside.shape, np.int64), "inside_bits": np.packbits(inside.reshape(-1)), "sigma": sigma,
              "pts_sha256": np.frombuffer(hashlib.sha256(np.ascontiguousarray(pts).tobytes()).hexdigest().encode(), np.uint8),
              "input_sha256": np.frombuffer(case_checksum(scene, masks).encode(), np.uint8)}
    np.savez_compressed(GOLDEN, **arrays)
    print("%s: grid %s, %d inside points, sigma in [%.2f, %.2f] -> %s (%d KB)" % (
        name, inside.shape, int(inside.sum()), float(sigma.min()), float(sigma.max()), GOLDEN, os.path.getsize(GOLDEN) // 1024))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    make_golden()
