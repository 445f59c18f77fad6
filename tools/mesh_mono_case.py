"""The People-Snapshot mesh dataset's case (TEST INFRASTRUCTURE ONLY): the monocular counterpart of oracle/mesh_case.py.

The scene is synth's body (scale 0.3 for the golden, 1.0 for the full-size frame) with the bounds of the monocular dataset's
`prepare_input` (lib/datasets/light_stage/monocular_dataset.py:32-71: y padded by 0.1 m), seen by one People-Snapshot
camera as `snapshot_data_utils.get_camera` builds it: K float64 from camera_f / camera_c, R = I, T = 0 and a non-zero
distortion D.  The mask is the body's silhouette with values 0 / 255; the image is noise (the mesh item does not read it).

    python -m tools.mesh_mono_case

(in the build container, where the reference tree exists) writes tests/golden/mesh_mono_s03.npz by running the UNMODIFIED
reference's `monocular_mesh_dataset.Dataset.__getitem__` on a stand-in `self` (vertices / params in a temp dir,
camera.pkl read by its own get_camera, imageio stubbed to return the synthetic jpg and png arrays).  It records the mask,
K, R and T that __getitem__ hands to `prepare_inside_pts`, and stores them with the reference's own `inside`, the cube's
sigma from the reference's `if_mesh_renderer.Renderer.render` and the sha256 of the inputs.  Existing golden files are not
touched.

`python -m tools.mesh_mono_case --drop-in OUT.npz` writes this package's drop-in item for the same frame (OpenCV's undistort
and resize, over a stand-in base class), so that tests can run it in a process of its own."""
import hashlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import mcubes_oracle, synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "mesh_mono_s03.npz")
RH, TH = (0.3, -0.2, 0.1), (0.1, 0.2, 1.0)     # synth.make_scene's defaults
RATIO = 0.5
# name -> (body scale, raw (pre-ratio) mask H, W, splat radius in raw pixels)
CASES = {
    "mono_s03": (0.3, 200, 150, 2),
    "mono_full": (1.0, 1080, 1080, 4),          # People-Snapshot's frame size; the item's mask is 540 x 540
}
CAMERA_K = np.array([-0.21, 0.09, 0.0015, -0.0011, 0.0])     # camera_k, the distortion D


def prepare_input(xyz_world, voxel_size):
    """monocular_dataset.py:32-71, literally; Rh = pose[:3] (3,), Th = trans (3,) float32."""
    xyz = np.asarray(xyz_world).astype(np.float32)
    min_xyz = np.min(xyz, axis=0)
    max_xyz = np.max(xyz, axis=0)
    min_xyz[1] -= 0.1
    max_xyz[1] += 0.1
    can_bounds = np.stack([min_xyz, max_xyz], axis=0)
    Rh = np.array(RH)
    R = synth._rodrigues(Rh).astype(np.float32)
    Th = np.array(TH).astype(np.float32)
    xyz = np.dot(xyz - Th, R)
    min_xyz = np.min(xyz, axis=0)
    max_xyz = np.max(xyz, axis=0)
    min_xyz[1] -= 0.1
    max_xyz[1] += 0.1
    bounds = np.stack([min_xyz, max_xyz], axis=0)
    dhw = xyz[:, [2, 1, 0]]
    min_dhw = min_xyz[[2, 1, 0]]
    max_dhw = max_xyz[[2, 1, 0]]
    voxel_size = np.array(voxel_size)
    coord = np.round((dhw - min_dhw) / voxel_size).astype(np.int32)
    out_sh = np.ceil((max_dhw - min_dhw) / voxel_size).astype(np.int32)
    out_sh = (out_sh | 31) + 1
    return coord, out_sh, can_bounds, bounds, Rh, Th


def make_scene(scale, seed=313, voxel_size=(0.005, 0.005, 0.005), num_train_frame=60):
    """synth's body and decoder with the monocular dataset's bounds: coord / out_sh / bounds / can_bounds / R / Th (B = 1,
    Th (1,3) as the monocular item's (3,) collates), volumes and weights built for this out_sh."""
    verts = synth.humanoid_vertices(seed, synth.N_SMPL_VERTS, scale)        # posed as synth.make_scene poses it
    world = (verts.astype(np.float64) @ synth._rodrigues(RH).T + np.asarray(TH, np.float64)).astype(np.float32)
    coord, out_sh, can_bounds, bounds, Rh, Th = prepare_input(world, voxel_size)
    volumes, _ = synth.make_volumes(coord, out_sh, seed)
    weights = synth.trained_like_rescale(synth.make_weights(seed, num_train_frame), volumes, seed)
    t = torch.from_numpy
    return {"coord": t(coord)[None], "out_sh": t(out_sh)[None], "bounds": t(bounds)[None], "can_bounds": t(can_bounds)[None],
            "R": t(synth._rodrigues(Rh).astype(np.float32))[None], "Th": t(Th)[None],
            "latent_index": torch.zeros(1, dtype=torch.int64), "volumes": volumes, "weights": weights,
            "voxel_size": [float(v) for v in voxel_size], "verts_world": t(world)}


def camera_pkl(scene, H, W):
    """The camera.pkl dict of a People-Snapshot subject: the body centred in an H x W frame, 80 % of its height."""
    cb = scene["can_bounds"][0].numpy().astype(np.float64)
    c = 0.5 * (cb[0] + cb[1])
    f = 0.8 * H * c[2] / (cb[1, 1] - cb[0, 1])
    return {"camera_f": np.array([f, f * 1.01]), "camera_c": np.array([W / 2.0 - f * c[0] / c[2] + 0.37,
                                                                        H / 2.0 - f * c[1] / c[2] - 0.21]),
            "camera_k": CAMERA_K.copy()}


def get_camera(pkl):
    """snapshot_data_utils.get_camera (:12-23) on the loaded pickle: K float64 on np.zeros([3, 3]), R = I, T = 0."""
    K = np.zeros([3, 3])
    K[0, 0] = pkl["camera_f"][0]
    K[1, 1] = pkl["camera_f"][1]
    K[:2, 2] = pkl["camera_c"]
    K[2, 2] = 1
    return {"K": K, "R": np.eye(3), "T": np.zeros([3]), "D": pkl["camera_k"]}


def silhouette(scene, K, H, W, radius, value=255):
    """The body's vertex cloud projected with K (R = I, T = 0) and splatted with discs: (H,W) uint8 of 0 / value."""
    uv = scene["verts_world"].numpy().astype(np.float64) @ K.T
    u = np.round(uv[:, 0] / uv[:, 2]).astype(int)
    v = np.round(uv[:, 1] / uv[:, 2]).astype(int)
    m = np.zeros((H, W), np.uint8)
    yy, xx = np.mgrid[-radius:radius + 1, -radius:radius + 1]
    disc = (yy ** 2 + xx ** 2) <= radius ** 2
    for dy, dx in zip(yy[disc], xx[disc]):
        uu, vv = u + dx, v + dy
        ok = (uu >= 0) & (uu < W) & (vv >= 0) & (vv < H)
        m[vv[ok], uu[ok]] = value
    return m


def build_case(name):
    """-> (scene, pkl, raw mask (H,W) uint8 0 / 255, raw image (H,W,3) uint8)."""
    scale, H, W, radius = CASES[name]
    scene = make_scene(scale)
    pkl = camera_pkl(scene, H, W)
    msk = silhouette(scene, get_camera(pkl)["K"], H, W, radius)
    img = np.random.RandomState(7).randint(0, 256, size=(H, W, 3)).astype(np.uint8)
    return scene, pkl, msk, img


def imread_stub(msk, img):
    """imageio.imread for the stand-in data root: image/<i>.jpg -> img, mask/<i>.png -> msk."""
    def imread(path):
        kind = os.path.basename(os.path.dirname(path))
        assert kind in ("image", "mask") and os.path.basename(path) == ("0.jpg" if kind == "image" else "0.png"), path
        return (img if kind == "image" else msk).copy()
    return imread


def stand_in_base(scene, pkl):
    """The reference Dataset's attributes as its __init__ / prepare_input leave them, for the synthetic frame."""
    world = scene["verts_world"].numpy()
    vs = scene["voxel_size"]

    class Base:
        def __init__(self):
            self.data_root = "synthetic"
            self.cam = get_camera(pkl)
            self.begin_ith_frame = 0
            self.num_train_frame = 1

        def prepare_input(self, i):
            return prepare_input(world, vs)

    return Base


def dropin_item(scene, pkl, msk, img, cv2=None):
    """This package's monocular drop-in item for frame 0 (cfg.ratio = RATIO)."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "datasets", "light_stage", "monocular_mesh_dataset.py")
    mod = load_source("neuralbody_b200.lib.datasets.light_stage.monocular_mesh_dataset", path)
    cfg.ratio = RATIO
    cls = mod.make_dataset_class(stand_in_base(scene, pkl), cv2=cv2, imread=imread_stub(msk, img))
    return cls()[0]


def case_checksum(scene, pkl, msk, img):
    """sha256 over everything the frame consumes (body, camera, raw mask and image, volumes, weights)."""
    h = hashlib.sha256()
    for k in ("coord", "out_sh", "bounds", "can_bounds", "R", "Th", "latent_index", "verts_world"):
        h.update(scene[k].contiguous().numpy().tobytes())
    for k in ("camera_f", "camera_c", "camera_k"):
        h.update(np.ascontiguousarray(pkl[k], np.float64).tobytes())
    h.update(msk.tobytes()); h.update(img.tobytes())
    for v in scene["volumes"]:
        h.update(v.contiguous().numpy().tobytes())
    for k in sorted(scene["weights"]):
        h.update(scene["weights"][k].contiguous().numpy().tobytes())
    return h.hexdigest()


def load_golden(path=GOLDEN):
    """-> dict: shape, inside (X,Y,Z) uint8 (mask values), sigma (n_inside,) float32, msk (H,W) uint8, K (3,3) / R (3,3) /
    T (3,1) float64 as prepare_inside_pts received them, pts_sha256, input_sha256, cube (padded float64, rebuilt)."""
    z = np.load(path)
    out = {k: z[k] for k in ("inside", "sigma", "msk", "K", "R", "T")}
    out["shape"] = out["inside"].shape
    out["pts_sha256"] = bytes(z["pts_sha256"]).decode()
    out["input_sha256"] = bytes(z["input_sha256"]).decode()
    out["cube"] = mcubes_oracle.pad_cube(out["inside"] != 0, out["sigma"].astype(np.float64))
    return out


def mesh_inside_f64(pts, K, R, T, msk):
    """monocular_mesh_dataset.py:35-48 (prepare_inside_pts with base_utils.project), literally: one view, numpy's own
    promotion of the float32 grid by the float64 camera."""
    sh = pts.shape
    pts3d = pts.reshape(-1, 3)
    RT = np.concatenate([R, T], axis=1)
    xyz = np.dot(pts3d, RT[:, :3].T) + RT[:, 3:].T
    xyz = np.dot(xyz, K.T)
    pts2d = xyz[:, :2] / xyz[:, 2:]
    H, W = msk.shape
    pts2d = np.round(pts2d).astype(np.int32)
    pts2d[:, 0] = np.clip(pts2d[:, 0], 0, W - 1)
    pts2d[:, 1] = np.clip(pts2d[:, 1], 0, H - 1)
    return msk[pts2d[:, 1], pts2d[:, 0]].reshape(*sh[:-1])


# ----------------------------------------------------------------------------- generator (needs the reference tree)
def _reference_item(scene, pkl, msk, img):
    """The reference's monocular_mesh_dataset.Dataset.__getitem__(0) on a stand-in `self`; -> (item, the arguments its
    prepare_inside_pts received)."""
    import pickle
    import tempfile
    import types
    from oracle import ref_harness
    cfg = ref_harness.load_reference()[0]
    for name in ("trimesh", "imageio", "plyfile"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.PlyData = object
            sys.modules[name] = m
    from lib.datasets.light_stage import monocular_mesh_dataset as ref_mono
    from lib.utils import snapshot_data_utils
    seen = {}
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "vertices"))
        np.save(os.path.join(d, "vertices", "0.npy"), scene["verts_world"].numpy())
        with open(os.path.join(d, "camera.pkl"), "wb") as f:
            pickle.dump(pkl, f)
        cam = snapshot_data_utils.get_camera(os.path.join(d, "camera.pkl"))
        mine = get_camera(pkl)
        assert all(np.array_equal(cam[k], mine[k]) and cam[k].dtype == mine[k].dtype for k in ("K", "R", "T", "D"))
        cfg.voxel_size = [float(v) for v in scene["voxel_size"]]
        cfg.ratio = RATIO
        pose = np.zeros((1, 72)); pose[0, :3] = RH
        fake = types.SimpleNamespace(data_root=d, cam=cam, begin_ith_frame=0, num_train_frame=1,
                                     params={"pose": pose, "trans": np.array([TH])})
        fake.prepare_input = lambda i: ref_mono.Dataset.prepare_input(fake, i)

        def prepare_inside_pts(pts, m, K, R, T):
            seen.update(pts=pts, msk=m.copy(), K=K.copy(), R=R.copy(), T=T.copy())
            return ref_mono.Dataset.prepare_inside_pts(fake, pts, m, K, R, T)

        fake.prepare_inside_pts = prepare_inside_pts
        old = ref_mono.imageio
        ref_mono.imageio = types.SimpleNamespace(imread=imread_stub(msk, img))
        try:
            item = ref_mono.Dataset.__getitem__(fake, 0)
        finally:
            ref_mono.imageio = old
    assert np.array_equal(item["out_sh"], scene["out_sh"][0].numpy()) and np.array_equal(item["coord"], scene["coord"][0].numpy())
    assert np.array_equal(item["bounds"], scene["bounds"][0].numpy())
    assert np.allclose(scene["R"][0].numpy(), item["R"], atol=1e-6) and np.array_equal(item["Th"], scene["Th"][0].numpy())
    return item, seen


def make_golden(name="mono_s03"):
    from torch.utils.data import default_collate
    from oracle import mesh_case
    scene, pkl, msk, img = build_case(name)
    item, seen = _reference_item(scene, pkl, msk, img)
    # the dtypes this case exists for: a float32 grid box and a float64 camera
    cb = prepare_input(scene["verts_world"].numpy(), scene["voxel_size"])[2]
    assert cb.dtype == np.float32 and np.array_equal(cb, scene["can_bounds"][0].numpy())
    assert all(seen[k].dtype == np.float64 for k in ("K", "R", "T")) and seen["msk"].dtype == np.uint8
    assert seen["msk"].shape == (int(msk.shape[0] * RATIO), int(msk.shape[1] * RATIO))
    pts, inside = item["pts"], item["inside"]
    assert pts.dtype == np.float32 and np.array_equal(pts, mesh_case.mesh_grid(cb, scene["voxel_size"]))
    assert np.array_equal(inside, mesh_inside_f64(pts, seen["K"], seen["R"], seen["T"], seen["msk"]))
    assert len(np.unique(inside)) > 2, np.unique(inside)        # 0, 255 and undistortion's in-between values
    batch = default_collate([{k: item[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}])
    batch["pts"], batch["inside"] = torch.from_numpy(pts)[None], torch.from_numpy(inside)[None]
    cube = mesh_case._reference_cube(scene, batch)
    assert cube.dtype == np.float64 and cube.shape == tuple(s + 20 for s in inside.shape)
    core = cube[10:-10, 10:-10, 10:-10]
    sigma = core[inside != 0].astype(np.float32)
    assert np.array_equal(sigma.astype(np.float64), core[inside != 0])
    arrays = {"inside": inside, "sigma": sigma, "msk": seen["msk"], "K": seen["K"], "R": seen["R"], "T": seen["T"],
              "pts_sha256": np.frombuffer(hashlib.sha256(np.ascontiguousarray(pts).tobytes()).hexdigest().encode(), np.uint8),
              "input_sha256": np.frombuffer(case_checksum(scene, pkl, msk, img).encode(), np.uint8)}
    np.savez_compressed(GOLDEN, **arrays)
    print("%s: grid %s, %d inside points (values %s), mask %s, sigma in [%.2f, %.2f] -> %s (%d KB)" % (
        name, inside.shape, int((inside != 0).sum()), np.unique(inside)[:6].tolist(), seen["msk"].shape, float(sigma.min()),
        float(sigma.max()), GOLDEN, os.path.getsize(GOLDEN) // 1024))


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--drop-in":
        it = dropin_item(*build_case("mono_s03"))
        np.savez(sys.argv[2], **{k: np.asarray(v) for k, v in it.items()})
    else:
        make_golden()
