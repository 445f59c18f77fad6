"""The demo datasets' camera rays (TEST INFRASTRUCTURE ONLY): a numpy restatement of upstream's per-view ray generation and
the generator of its goldens.

`image_rays_numpy(RT, K, bounds, H, W)` restates render_utils.image_rays (lib/utils/render_utils.py:120-137): get_rays
(lib/utils/if_nerf/if_nerf_data_utils.py:8-21), `.astype(np.float32)`, get_near_far (:54-69) and the mask_at_box
compaction, with every rounding spelled out.  Upstream's three products go through numpy's `np.dot`, which hands them to
the BLAS; with numpy 2.3's OpenBLAS 0.3.30 (Haswell kernels) their arithmetic is, per output component:
  float64 camera (the multi-view demo sets)
    xy1 @ inv(K).T                   ddot:     fma(1, Ka2, fma(j, Ka1, i * Ka0))
    (pixel_camera - T) @ R           ddot:     fma(p2, R2a, fma(p1, R1a, p0 * R0a))
  float32 camera (the People-Snapshot demo)
    xy1 @ inv(K).T                   sdot, unit strides: the float products summed in double, rounded once
    (pixel_camera - T) @ R           sdot, R's stride 3: fma(p0, R0a, p1 * R1a) + p2 * R2a     (float)
Both fmas are emulated exactly (`fma64`, `fma32`).  The camera centre rays_o = -np.dot(R.T, T) is one gemv per view whose
rounding depends on R's memory layout (R sliced out of RT and a contiguous copy of it give different float32 bits), so it
is not restated: it is computed with upstream's own expression on upstream's own operands, as inv(K) is, and handed to the
kernel with it.  The GPU kernel (nb_image_rays / nb_image_rays_f64) carries the same
operations; the goldens below pin them to upstream's own output.

    python -m tools.demo_case

(in the build container, where the reference tree exists) writes, overwriting them, tests/golden/demo_mv_s64.npz and
demo_mono_s64.npz by running the UNMODIFIED reference's multi_view_demo_dataset / monocular_demo_dataset `__getitem__` on
small synthetic data directories (annots.npy with cams, vertices, params, mask PNGs; camera.pkl), with imageio / plyfile
stubbed, and tests/golden/demo_orbit_s512.npz, the full-size orbit cameras (`make_orbit`).  Each file holds the camera
and box image_rays received (and, for the first two, its outputs) with the sha256 of the synthetic inputs, which
`input_checksum` over `write_mv_root` / `write_mono_root` / `write_orbit_root` reproduces without the reference tree.

`upstream_image_rays` is the same computation as upstream writes it, with plain np.dot / np.linalg.norm and no rounding
spelled out: tools/bench_demo.py times it as upstream's host cost (it reproduces the goldens bit for bit as well)."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_MV = os.path.join(ROOT, "tests", "golden", "demo_mv_s64.npz")
GOLDEN_MONO = os.path.join(ROOT, "tests", "golden", "demo_mono_s64.npz")


# ----------------------------------------------------------------------------- exact fma in numpy
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = a * 134217729.0        # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _round_odd(s, e):
    """s + e (s = RN(s + e), the exact error e) rounded to odd."""
    odd = (s.view(np.int64) & 1) == 1
    step = np.nextafter(s, np.where(e > 0, np.inf, -np.inf))
    return np.where((e == 0) | odd, s, step)


def fma64(a, b, c):
    """Correctly rounded a * b + c in float64 (Boldo & Melquiond's emulation through rounding to odd)."""
    a, b, c = (np.asarray(x, dtype=np.float64) for x in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    v, ev = _two_sum(tl, ul)
    return (th + _round_odd(v, ev)).astype(np.float64)


def fma32(a, b, c):
    """Correctly rounded a * b + c in float32: the product is exact in float64, the sum rounded to odd there and then to
    float32 (53 >= 24 + 2 bits, so the two roundings are one)."""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    s, e = _two_sum(*np.broadcast_arrays(a * b, c))
    return _round_odd(s, e).astype(np.float32)


# ----------------------------------------------------------------------------- the restatement
def camera_centre(R, T):
    """rays_o of get_rays (:10), upstream's expression on the operands as upstream slices them from RT."""
    return -np.dot(R.T, T).ravel()


def get_rays_numpy(H, W, K_inv, R, T, o):
    """if_nerf_data_utils.get_rays with upstream's BLAS arithmetic (see the module doc).  K_inv = np.linalg.inv(K) in K's
    dtype; R (3,3), T (3,) and the camera centre o = camera_centre(R, T) in the camera's dtype.  -> ray_o (3,), ray_d
    (H*W,3), both in the camera's dtype."""
    f64 = R.dtype == np.float64
    dt = np.float64 if f64 else np.float32
    R, T, K_inv, o = (np.asarray(x, dtype=dt) for x in (R, T, K_inv, o))
    i, j = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    i, j = i.reshape(-1, 1).astype(dt), j.reshape(-1, 1).astype(dt)
    fma = fma64 if f64 else fma32
    if f64:
        pc = fma(1.0, K_inv[:, 2][None], fma(j, K_inv[:, 1][None], i * K_inv[:, 0][None]))
    else:
        w = [(x * K_inv[:, k][None]).astype(np.float64) for k, x in enumerate((i, j, np.ones_like(i)))]
        pc = ((w[0] + w[1]) + w[2]).astype(np.float32)
    p = pc - T[None]
    if f64:
        pw = fma(p[:, 2:3], R[2][None], fma(p[:, 1:2], R[1][None], p[:, 0:1] * R[0][None]))
    else:
        pw = fma(p[:, 0:1], R[0][None], p[:, 1:2] * R[1][None]) + p[:, 2:3] * R[2][None]
    return o.astype(dt), (pw - o[None]).astype(dt)


def image_rays_numpy(RT, K, bounds, H, W):
    """render_utils.image_rays restated: -> ray_o, ray_d (n,3), near, far (n,) float32 and mask_at_box (H*W,) bool."""
    RT, K = np.asarray(RT), np.asarray(K)
    if RT.dtype != K.dtype or RT.dtype not in (np.float32, np.float64):
        raise ValueError("RT and K must both be float32 or both float64")
    o, d = get_rays_numpy(int(H), int(W), np.linalg.inv(K), RT[:3, :3], RT[:3, 3], camera_centre(RT[:3, :3], RT[:3, 3]))
    ray_d = d.astype(np.float32)
    ray_o = np.broadcast_to(o.astype(np.float32), ray_d.shape)
    bounds = np.asarray(bounds, dtype=np.float32)
    # get_near_far, float32 throughout
    norm = np.sqrt((ray_d[:, 0] * ray_d[:, 0] + ray_d[:, 1] * ray_d[:, 1]) + ray_d[:, 2] * ray_d[:, 2])[:, None]
    v = ray_d / norm
    v[(v < np.float32(1e-5)) & (v > np.float32(-1e-10))] = np.float32(1e-5)
    v[(v > np.float32(-1e-5)) & (v < np.float32(1e-10))] = np.float32(-1e-5)
    tmin = (bounds[:1] - ray_o[:1]) / v
    tmax = (bounds[1:2] - ray_o[:1]) / v
    near = np.max(np.minimum(tmin, tmax), axis=-1)
    far = np.min(np.maximum(tmin, tmax), axis=-1)
    m = near < far
    return ray_o[m], ray_d[m], near[m] / norm[m, 0], far[m] / norm[m, 0], m


def upstream_image_rays(RT, K, bounds, H, W):
    """render_utils.image_rays as upstream computes it (get_rays, `.astype(np.float32)`, get_near_far, the compaction), with
    numpy's own np.dot and np.linalg.norm: what a view costs on the host.  -> ray_o, ray_d, near, far, mask_at_box."""
    R, T = RT[:3, :3], RT[:3, 3]
    centre = -np.dot(R.T, T).ravel()
    u, v = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    pix = np.stack([u, v, np.ones_like(u)], axis=2)
    world = np.dot(np.dot(pix, np.linalg.inv(K).T) - T.ravel(), R)
    ray_d = (world - centre[None, None]).reshape(-1, 3).astype(np.float32)
    ray_o = np.broadcast_to(centre, world.shape).reshape(-1, 3).astype(np.float32)
    norm = np.linalg.norm(ray_d, axis=-1, keepdims=True)
    vd = ray_d / norm
    vd[(vd < 1e-5) & (vd > -1e-10)] = 1e-5
    vd[(vd > -1e-5) & (vd < 1e-10)] = -1e-5
    lo = (bounds[:1] - ray_o[:1]) / vd
    hi = (bounds[1:2] - ray_o[:1]) / vd
    near = np.max(np.minimum(lo, hi), axis=-1)
    far = np.min(np.maximum(lo, hi), axis=-1)
    m = near < far
    return (ray_o[m], ray_d[m], (near[m] / norm[m, 0]).astype(np.float32), (far[m] / norm[m, 0]).astype(np.float32), m)


# ----------------------------------------------------------------------------- synthetic demo data
RATIO = 0.5
RAW_HW = (128, 96)              # cfg.H, cfg.W: the item's views are 64 x 48 (H != W)
MV_VIEWS = (0, 37, 90)          # gen_path views of the 144-view orbit kept in the golden
MONO_VIEWS = (0, 50)            # monocular orbit angles (of 144)
DIST = np.array([-0.21, 0.09, 0.0015, -0.0011, 0.0])


def body_vertices(seed=313, n=6890):
    """A body-sized point cloud in the world (metres, y down as in ZJU-MoCap's world): an ellipsoid shell."""
    rng = np.random.RandomState(seed)
    u = rng.randn(n, 3)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    return (u * np.array([0.25, 0.85, 0.15]) + np.array([0.05, -0.1, 0.02])).astype(np.float32)


def ring_cams(nv=4, radius=3.0, H=RAW_HW[0], W=RAW_HW[1]):
    """annots['cams'] of nv cameras on a ring around the body, looking at it: K, R, D lists and T in millimetres."""
    import cv2
    cams = {"K": [], "R": [], "T": [], "D": []}
    for v in range(nv):
        a = 2 * np.pi * v / nv + 0.1
        c = np.array([radius * np.sin(a), -0.3, radius * np.cos(a)])
        z = -c / np.linalg.norm(c)
        x = np.cross(np.array([0., 1., 0.]), z); x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])
        R = cv2.Rodrigues(cv2.Rodrigues(R)[0])[0]
        f = 1.1 * H
        cams["K"].append(np.array([[f, 0, W / 2 + 0.3 * v], [0, f * 1.01, H / 2 - 0.2], [0, 0, 1]]))
        cams["R"].append(R)
        cams["T"].append((-R @ c)[:, None] * 1000.)
        cams["D"].append(DIST[:, None] * (1 + 0.1 * v))
    return cams


def silhouette(verts, K, R, T, H, W, value=255):
    """The vertex cloud projected into one raw view, splatted 2 px wide: (H,W) uint8 of 0 / value."""
    uv = (verts.astype(np.float64) @ R.T + T.reshape(1, 3)) @ K.T
    u = np.round(uv[:, 0] / uv[:, 2]).astype(int)
    v = np.round(uv[:, 1] / uv[:, 2]).astype(int)
    m = np.zeros((H, W), np.uint8)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            ok = (u + dx >= 0) & (u + dx < W) & (v + dy >= 0) & (v + dy < H)
            m[v[ok] + dy, u[ok] + dx] = value
    return m


def write_mv_root(d, nv=4, n_frames=2):
    """A ZJU-MoCap-like data root: annots.npy (cams, ims), vertices/<i>.npy, params/<i>.npy, mask_cihp/<view>/<i>.png
    contents kept in a dict (the PNG reader is stubbed: no image codec needed) -> {mask path: array}."""
    cams = ring_cams(nv)
    verts = body_vertices()
    ims = [{"ims": ["Camera_B%d/%06d.jpg" % (v + 1, i) for v in range(nv)]} for i in range(n_frames)]
    np.save(os.path.join(d, "annots.npy"), {"cams": cams, "ims": ims}, allow_pickle=True)
    masks = {}
    for sub in ("vertices", "params"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    for i in range(n_frames):
        vi = verts + np.float32(0.01 * i)
        np.save(os.path.join(d, "vertices", "%d.npy" % i), vi)
        np.save(os.path.join(d, "params", "%d.npy" % i), {"Rh": np.array([[0.1, 0.2 + 0.05 * i, -0.05]]),
                                                           "Th": np.array([[0.05, -0.1, 0.02]])}, allow_pickle=True)
        for v in range(nv):
            T = np.asarray(cams["T"][v]) / 1000.
            masks[os.path.join(d, "mask_cihp", ims[i]["ims"][v])[:-4] + ".png"] = silhouette(
                vi, np.asarray(cams["K"][v]), np.asarray(cams["R"][v]), T, RAW_HW[0], RAW_HW[1])
    return masks


def camera_pkl(H=RAW_HW[0], W=RAW_HW[1]):
    """A People-Snapshot camera.pkl: the body 2.6 m in front of the camera."""
    f = 1.2 * H
    return {"camera_f": np.array([f, f * 1.01]), "camera_c": np.array([W / 2.0 + 0.37, H / 2.0 - 0.21]),
            "camera_k": DIST.copy()}


def write_mono_root(d):
    """A People-Snapshot-like data root: camera.pkl, vertices/0.npy, the params dict (pose, trans) -> (params path,
    {mask path: array})."""
    import pickle
    verts = body_vertices(seed=7) + np.array([0., 0., 2.6], np.float32)
    os.makedirs(os.path.join(d, "vertices"), exist_ok=True)
    np.save(os.path.join(d, "vertices", "0.npy"), verts)
    pkl = camera_pkl()
    with open(os.path.join(d, "camera.pkl"), "wb") as f:
        pickle.dump(pkl, f)
    pose = np.zeros((1, 72)); pose[0, :3] = (0.1, 0.3, -0.05)
    params = os.path.join(d, "params.npy")
    np.save(params, {"pose": pose, "trans": np.array([[0.0, 0.05, 2.6]])}, allow_pickle=True)
    K = np.array([[pkl["camera_f"][0], 0, pkl["camera_c"][0]], [0, pkl["camera_f"][1], pkl["camera_c"][1]], [0, 0, 1.]])
    return params, {os.path.join(d, "mask", "0.png"): silhouette(verts, K, np.eye(3), np.zeros(3), RAW_HW[0], RAW_HW[1])}


def input_checksum(d, masks):
    """sha256 over every file of the data root and the stubbed mask images, in sorted order."""
    h = hashlib.sha256()
    for root, _, files in sorted(os.walk(d)):
        for f in sorted(files):
            with open(os.path.join(root, f), "rb") as fh:
                h.update(fh.read())
    for k in sorted(masks):
        h.update(masks[k].tobytes())
    return h.hexdigest()


# ----------------------------------------------------------------------------- generator (needs the reference tree)
def _reference_setup(num_render_views=144):
    import types
    from oracle import ref_harness
    cfg = ref_harness.load_reference()[0]
    for name in ("trimesh", "imageio", "plyfile"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.PlyData = object
            sys.modules[name] = m
    cfg.ratio, cfg.H, cfg.W = RATIO, RAW_HW[0], RAW_HW[1]
    cfg.num_render_views, cfg.num_train_frame, cfg.begin_ith_frame, cfg.ith_frame = num_render_views, 2, 0, 0
    cfg.training_view, cfg.frame_interval, cfg.big_box = [0, 1, 2, 3], 1, False
    cfg.vertices, cfg.params, cfg.num_render_frame = "vertices", "params", -1
    cfg.voxel_size = [0.005, 0.005, 0.005]
    return cfg


def _run_items(mod, ds, masks, views):
    """mod.Dataset.__getitem__ over `views` with imageio stubbed and render_utils.image_rays recorded -> [(item, call)]."""
    import types
    calls = []
    orig = mod.render_utils.image_rays

    def image_rays(RT, K, bounds):
        out = orig(RT, K, bounds)
        calls.append({"RT": np.array(RT), "K": np.array(K), "bounds": np.array(bounds), "out": out})
        return out

    old_io, old_ir = mod.imageio, mod.render_utils.image_rays
    mod.imageio = types.SimpleNamespace(imread=lambda p: masks[p].copy())
    mod.render_utils.image_rays = image_rays
    try:
        items = [ds[v] for v in views]
    finally:
        mod.imageio, mod.render_utils.image_rays = old_io, old_ir
    return list(zip(items, calls))


def reference_items(kind, views, d):
    """The UNMODIFIED reference dataset `kind` ('mv' = multi_view_demo_dataset, 'perform' = multi_view_perform_dataset,
    'mono' = monocular_demo_dataset) built on a synthetic root in `d` -> ([(item, image_rays call)], input sha256)."""
    _reference_setup()
    if kind == "mono":
        from lib.datasets.light_stage import monocular_demo_dataset as mod
        params, masks = write_mono_root(d)
        ds = mod.Dataset(d, "synthetic", params, "test")
    else:
        if kind == "mv":
            from lib.datasets.light_stage import multi_view_demo_dataset as mod
        else:
            from lib.datasets.light_stage import multi_view_perform_dataset as mod
        masks = write_mv_root(d)
        ds = mod.Dataset(d, "synthetic", os.path.join(d, "annots.npy"), "test")
    return _run_items(mod, ds, masks, views), input_checksum(d, masks), ds, masks


def make_golden(kind, views, path):
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        pairs, sha, _, _ = reference_items(kind, views, d)
    arrays = {"input_sha256": np.frombuffer(sha.encode(), np.uint8), "H": np.array(int(RAW_HW[0] * RATIO)),
              "W": np.array(int(RAW_HW[1] * RATIO))}
    for v, (item, call) in zip(views, pairs):
        ray_o, ray_d, near, far, _, _, mask = call["out"]
        mine = image_rays_numpy(call["RT"], call["K"], call["bounds"], arrays["H"], arrays["W"])
        assert all(np.array_equal(a, b) for a, b in zip((ray_o, ray_d, near, far, mask), mine)), "restatement differs"
        assert 0 < mask.sum() < mask.size
        for k, x in (("RT", call["RT"]), ("K", call["K"]), ("bounds", call["bounds"]), ("ray_o", ray_o), ("ray_d", ray_d),
                     ("near", near), ("far", far), ("mask_at_box", mask)):
            arrays["%s_%d" % (k, v)] = x
    arrays["views"] = np.array(views)
    np.savez_compressed(path, **arrays)
    print("%s: views %s, n = %s, camera %s -> %s (%d KB)" % (kind, views, [int(arrays["mask_at_box_%d" % v].sum()) for v in views],
                                                          arrays["RT_%d" % views[0]].dtype, path, os.path.getsize(path) // 1024))


def load_golden(path):
    z = np.load(path)
    views = [int(v) for v in z["views"]]
    out = {"H": int(z["H"]), "W": int(z["W"]), "input_sha256": bytes(z["input_sha256"]).decode(), "views": {}}
    for v in views:
        out["views"][v] = {k: z["%s_%d" % (k, v)] for k in ("RT", "K", "bounds", "ray_o", "ray_d", "near", "far", "mask_at_box")}
    return out


ORBIT = os.path.join(ROOT, "tests", "golden", "demo_orbit_s512.npz")
ORBIT_MV_VIEWS = (0, 23, 61, 102, 140)
ORBIT_MONO_VIEWS = (0, 36, 72, 108)


def write_orbit_root(d):
    """The full-size orbit's inputs: annots.npy with four 1024 x 1024 ring cameras, and a People-Snapshot root (vertices,
    params) with a 1080 x 1080 camera.pkl -> (params path, {mask path: array})."""
    import pickle
    np.save(os.path.join(d, "annots.npy"), {"cams": ring_cams(4, H=1024, W=1024), "ims": []}, allow_pickle=True)
    params, masks = write_mono_root(d)
    with open(os.path.join(d, "camera.pkl"), "wb") as f:
        pickle.dump(camera_pkl(1080, 1080), f)
    return params, masks


def make_orbit(path=ORBIT):
    """Full-size cameras for the restatement tests: five views of the 144-view gen_path orbit around four ZJU-MoCap-like
    1024 x 1024 cameras (512 x 512 renders, float64) and four angles of the People-Snapshot orbit (1080 x 1080 -> 540 x 540,
    float32 camera, the rotated body's can_bounds), all from the reference's own code."""
    import tempfile
    cfg = _reference_setup()
    cfg.H = cfg.W = 1024
    from lib.utils import render_utils
    from lib.datasets.light_stage import monocular_demo_dataset as mono
    with tempfile.TemporaryDirectory() as d:
        params, masks = write_orbit_root(d)
        sha = input_checksum(d, masks)
        K, RT = render_utils.load_cam(os.path.join(d, "annots.npy"))
        w2c = render_utils.gen_path(RT)
        verts = body_vertices()
        mn, mx = verts.min(0), verts.max(0)
        mn[2] -= 0.05; mx[2] += 0.05
        arrays = {"mv_RT": np.stack([w2c[v] for v in ORBIT_MV_VIEWS]), "mv_K": K[0], "mv_bounds": np.stack([mn, mx]),
                  "mv_views": np.array(ORBIT_MV_VIEWS), "mv_HW": np.array([512, 512])}
        cfg.ratio = RATIO
        ds = mono.Dataset(d, "synthetic", params, "test")
        Km = ds.cam["K"].copy().astype(np.float32)
        Km[:2] = Km[:2] * cfg.ratio
        arrays.update({"mono_RT": np.concatenate([ds.cam["R"], ds.cam["T"][:, None]], axis=1).astype(np.float32),
                       "mono_K": Km, "mono_bounds": np.stack([ds.prepare_input(0, v)[2] for v in ORBIT_MONO_VIEWS]),
                       "mono_views": np.array(ORBIT_MONO_VIEWS), "mono_HW": np.array([540, 540]),
                       "input_sha256": np.frombuffer(sha.encode(), np.uint8)})
    assert arrays["mv_RT"].dtype == np.float64 and arrays["mono_RT"].dtype == np.float32
    assert arrays["mv_bounds"].dtype == np.float32 and arrays["mono_bounds"].dtype == np.float32
    for k in ("mv", "mono"):
        H, W = arrays[k + "_HW"]
        for j in range(len(arrays[k + "_views"])):
            RT = arrays[k + "_RT"][j] if k == "mv" else arrays["mono_RT"]
            b = arrays["mv_bounds"] if k == "mv" else arrays["mono_bounds"][j]
            n = int(image_rays_numpy(RT, arrays[k + "_K"], b, H, W)[4].sum())
            assert 1000 < n < H * W, (k, j, n)
    np.savez_compressed(path, **arrays)
    print("orbit cameras -> %s" % path)


if __name__ == "__main__":
    make_golden("mv", MV_VIEWS, GOLDEN_MV)
    make_golden("mono", MONO_VIEWS, GOLDEN_MONO)
    make_orbit()
