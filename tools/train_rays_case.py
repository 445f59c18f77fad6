"""The training datasets' sampled rays (TEST INFRASTRUCTURE ONLY): a numpy restatement of upstream's training item and the
generator of its goldens.

`sample_numpy(...)` restates if_nerf_data_utils.sample_ray_h36m / sample_ray, split 'train' (:153-219 / :72-137), given
the class map (neuralbody_b200.lib.datasets.train_item) and upstream's np.random.randint results: the rounds, get_rays at
each candidate pixel with the BLAS roundings tools/demo_case.py spells out (K's product in K's dtype, then float64), and
get_near_far in float64.  `upstream_sample(...)` is the same item as upstream computes it, with numpy's own get_rays over the
whole image, np.argwhere and np.random.randint: what an item costs on the host (tools/bench_train_data.py times it).

    python -m tools.train_rays_case

(in the build container, where the reference tree exists) writes, overwriting them, tests/golden/train_rays_mv.npz and
train_rays_mono.npz by running the UNMODIFIED reference's multi_view_dataset / monocular_dataset `__getitem__` (split
'train') on small synthetic data roots (demo_case's, plus images), with imageio stubbed and np.random.randint wrapped to
record every draw.  Each case holds what the sampler received (the processed image, mask, camera, box, N_rand, ratios), the
class map, the draws, the rounds and upstream's outputs, with the sha256 of the synthetic inputs; and one split-'test' item
(`test_*`: what the sampler received and every box-hit ray of the view with its colour)."""
import contextlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools import demo_case as DC  # noqa: E402
from neuralbody_b200.lib.datasets import train_item  # noqa: E402

GOLDEN_MV = os.path.join(ROOT, "tests", "golden", "train_rays_mv.npz")
GOLDEN_MONO = os.path.join(ROOT, "tests", "golden", "train_rays_mono.npz")
# (index, N_rand, body_sample_ratio, face_sample_ratio, label-13 pixels in the mask)
# (cases 0 and 4 of each share N_rand and the ratios over different views / masks: the two-item batches of the GPU test)
MV_CASES = ((0, 1000, 0.5, 0.0, False), (1, 3000, 0.5, 0.2, False), (2, 1000, 0.3, 0.0, False), (3, 777, 0.5, 0.0, False),
            (1, 1000, 0.5, 0.0, False))
MONO_CASES = ((0, 1000, 0.5, 0.2, False), (0, 3000, 0.5, 0.2, True), (0, 1000, 0.4, 0.3, True), (0, 1000, 0.4, 0.3, True),
              (0, 1000, 0.5, 0.2, True))
TEST_INDEX = 0                  # the split-'test' item of each golden


# ----------------------------------------------------------------------------- the restatement
def camera_rays_numpy(K_inv, R, T, o, ys, xs):
    """get_rays (:8-21) at the pixels (ys, xs), float64 R / T / o, K_inv in K's dtype -> ray_d (n,3) float64."""
    i, j = xs.astype(np.float32)[:, None], ys.astype(np.float32)[:, None]
    if K_inv.dtype == np.float64:
        i, j = i.astype(np.float64), j.astype(np.float64)
        pc = DC.fma64(1.0, K_inv[:, 2][None], DC.fma64(j, K_inv[:, 1][None], i * K_inv[:, 0][None]))
    else:
        w = [(x * K_inv[:, k][None]).astype(np.float64) for k, x in enumerate((i, j, np.ones_like(i)))]
        pc = ((w[0] + w[1]) + w[2]).astype(np.float32).astype(np.float64)
    p = pc - T.reshape(1, 3)
    pw = DC.fma64(p[:, 2:3], R[2][None], DC.fma64(p[:, 1:2], R[1][None], p[:, 0:1] * R[0][None]))
    return pw - o[None]


def near_far64(o, d, bounds):
    """get_near_far (:54-69) on float64 rays, the float32 box promoted -> near, far (float64, before the division) and the
    norm."""
    norm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]
    v = d / norm
    v[(v < 1e-5) & (v > -1e-10)] = 1e-5
    v[(v > -1e-5) & (v < 1e-10)] = -1e-5
    b = bounds.astype(np.float64)
    tmin, tmax = (b[:1] - o[None]) / v, (b[1:2] - o[None]) / v
    return np.max(np.minimum(tmin, tmax), axis=-1), np.min(np.maximum(tmin, tmax), axis=-1), norm[:, 0]


def sample_numpy(img, class_map, K, R, T, bounds, n_rays, body_ratio, face_ratio, draws, rng=None):
    """The training item's rays from upstream's draws (one flat int64 array, rounds in order; or, with `rng`, drawn from
    rng.randint as upstream draws them) -> rgb, ray_o, ray_d, near, far (float32), coord (n,2), the number of rounds and
    the draws."""
    if rng is not None:
        drawn, draws = [], np.zeros(0, np.int64)
    K_inv = np.linalg.inv(K)
    o = -np.dot(R.T, T).ravel()
    lists = [np.argwhere(class_map & bit) for bit in (train_item.BODY, train_item.FACE, train_item.BOUND)]
    out, sampled, cur, rounds = [], 0, 0, 0
    while sampled < n_rays:
        m = n_rays - sampled
        n_body, n_face = int(m * body_ratio), int(m * face_ratio)
        sizes = (n_body, n_face if len(lists[1]) else 0, m - n_body - n_face)
        coord = []
        for lst, n in zip(lists, sizes):
            if rng is not None and n:
                drawn.append(rng.randint(0, len(lst), n))
                draws = np.concatenate(drawn)
            coord.append(lst[draws[cur:cur + n]])
            cur += n
        coord = np.concatenate(coord)
        d = camera_rays_numpy(K_inv, R, T, o, coord[:, 0], coord[:, 1])
        near, far, norm = near_far64(o, d, bounds)
        hit = near < far
        out.append((coord[hit], d[hit], near[hit] / norm[hit], far[hit] / norm[hit]))
        sampled += int(hit.sum())
        rounds += 1
    assert cur == len(draws), "draws left over"
    coord = np.concatenate([c[0] for c in out])
    d = np.concatenate([c[1] for c in out]).astype(np.float32)
    return (img[coord[:, 0], coord[:, 1]].astype(np.float32), np.broadcast_to(o.astype(np.float32), d.shape).copy(), d,
            np.concatenate([c[2] for c in out]).astype(np.float32), np.concatenate([c[3] for c in out]).astype(np.float32),
            coord, rounds, np.asarray(draws, np.int64))


def upstream_sample(img, class_map, K, R, T, bounds, n_rays, body_ratio, face_ratio):
    """The training item's rays as upstream computes them (float64 get_rays over the whole image with numpy's own np.dot,
    np.argwhere per list and round, np.random.randint, get_near_far): the host cost of upstream's sampler."""
    H, W = img.shape[:2]
    o = -np.dot(R.T, T).ravel()
    u, v = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32), indexing='xy')
    world = np.dot(np.dot(np.stack([u, v, np.ones_like(u)], axis=2), np.linalg.inv(K).T) - T.ravel(), R)
    ray_d_all = world - o[None, None]
    parts, sampled = [], 0
    while sampled < n_rays:
        m = n_rays - sampled
        n_body, n_face = int(m * body_ratio), int(m * face_ratio)
        body = np.argwhere(class_map & train_item.BODY)
        body = body[np.random.randint(0, len(body), n_body)]
        face = np.argwhere(class_map & train_item.FACE)
        if len(face) > 0:
            face = face[np.random.randint(0, len(face), n_face)]
        bound = np.argwhere(class_map & train_item.BOUND)
        bound = bound[np.random.randint(0, len(bound), m - n_body - n_face)]
        coord = np.concatenate([body, face, bound] if len(face) else [body, bound])
        d = ray_d_all[coord[:, 0], coord[:, 1]]
        norm = np.linalg.norm(d, axis=-1, keepdims=True)
        vd = d / norm
        vd[(vd < 1e-5) & (vd > -1e-10)] = 1e-5
        vd[(vd > -1e-5) & (vd < 1e-10)] = -1e-5
        lo, hi = (bounds[:1] - o[None]) / vd, (bounds[1:2] - o[None]) / vd
        near, far = np.max(np.minimum(lo, hi), axis=-1), np.min(np.maximum(lo, hi), axis=-1)
        hit = near < far
        parts.append((d[hit], img[coord[hit, 0], coord[hit, 1]], near[hit] / norm[hit, 0], far[hit] / norm[hit, 0]))
        sampled += int(hit.sum())
    d = np.concatenate([p[0] for p in parts]).astype(np.float32)
    return (np.concatenate([p[1] for p in parts]).astype(np.float32), np.broadcast_to(o, d.shape).astype(np.float32), d,
            np.concatenate([p[2] for p in parts]).astype(np.float32), np.concatenate([p[3] for p in parts]).astype(np.float32))


# ----------------------------------------------------------------------------- synthetic training data
def body_image(mask, seed):
    """An RGB uint8 image: a smooth colour field with noise, brighter on the silhouette."""
    rng = np.random.RandomState(seed)
    H, W = mask.shape
    y, x = np.mgrid[0:H, 0:W]
    img = np.stack([(x * 255) // W, (y * 255) // H, (x + y) % 256], axis=-1).astype(np.int32)
    img += rng.randint(0, 40, size=img.shape) + (mask[..., None] > 0) * 60
    return np.clip(img, 0, 255).astype(np.uint8)


def add_face(mask):
    """Label 13 (CIHP's face) on the top part of the silhouette."""
    m = mask.copy()
    ys = np.nonzero(m.any(axis=1))[0]
    top = ys[:max(1, len(ys) // 6)]
    m[top] = np.where(m[top] > 0, 13, 0)
    return m


def write_mv_train_root(d):
    """demo_case.write_mv_root plus one image per mask -> {path: array} of every stubbed image read."""
    files = DC.write_mv_root(d)
    for k, m in list(files.items()):
        files[k.replace(os.path.join(d, "mask_cihp") + os.sep, d + os.sep)[:-4] + ".jpg"] = body_image(m, len(files))
    return files


def write_mono_train_root(d):
    """demo_case.write_mono_root plus image/0.jpg, and the mask with label-13 pixels under mask13/ -> (params, files)."""
    params, files = DC.write_mono_root(d)
    m = files[os.path.join(d, "mask", "0.png")]
    files[os.path.join(d, "image", "0.jpg")] = body_image(m, 7)
    files[os.path.join(d, "mask13", "0.png")] = add_face(m)
    return params, files


def input_checksum(d, files):
    return DC.input_checksum(d, files)


# ----------------------------------------------------------------------------- generator (needs the reference tree)
@contextlib.contextmanager
def recorded(mod, files, alias=None):
    """imageio stubbed to `files` (alias: path -> path it reads instead), np.random.randint and the module's sampler wrapped
    to record every draw and call."""
    import types
    rec = {"draws": [], "calls": []}
    orig_randint = np.random.randint
    name = "sample_ray_h36m" if hasattr(mod, "Dataset") and mod.__name__.endswith("multi_view_dataset") else "sample_ray"
    orig_sampler = getattr(mod.if_nerf_dutils, name)

    def randint(*a, **k):
        r = orig_randint(*a, **k)
        rec["draws"].append(np.asarray(r, np.int64).ravel())
        return r

    def sampler(img, msk, K, R, T, bounds, nrays, split):
        rec["draws"].clear()
        out = orig_sampler(img, msk, K, R, T, bounds, nrays, split)
        rec["calls"].append({"img": img.copy(), "msk": msk.copy(), "K": K.copy(), "R": R.copy(), "T": T.copy(),
                             "bounds": bounds.copy(), "nrays": nrays, "out": out, "draws": list(rec["draws"])})
        return out

    old = mod.imageio
    mod.imageio = types.SimpleNamespace(imread=lambda p: files[(alias or {}).get(p, p)].copy())
    np.random.randint = randint
    setattr(mod.if_nerf_dutils, name, sampler)
    try:
        yield rec
    finally:
        mod.imageio = old
        np.random.randint = orig_randint
        setattr(mod.if_nerf_dutils, name, orig_sampler)


def reference_setup():
    cfg = DC._reference_setup()
    cfg.mask_bkgd, cfg.white_bkgd, cfg.test_novel_pose = True, False, False
    return cfg


def reference_items(kind, cases, d, split="train"):
    """The UNMODIFIED reference training dataset `kind` ('mv', 'mono') for `split` on a synthetic root in `d`, one item per
    case -> ([(item, sampler call)], sha256, dataset, files)."""
    cfg = reference_setup()
    if kind == "mv":
        from lib.datasets.light_stage import multi_view_dataset as mod
        files = write_mv_train_root(d)
        ds = mod.Dataset(d, "synthetic", os.path.join(d, "annots.npy"), split)
    else:
        from lib.datasets.light_stage import monocular_dataset as mod
        params, files = write_mono_train_root(d)
        ds = mod.Dataset(d, "synthetic", params, split)
    pairs = []
    for c, (index, nrays, rb, rf, face) in enumerate(cases):
        cfg.body_sample_ratio, cfg.face_sample_ratio = rb, rf
        ds.nrays = nrays
        alias = {os.path.join(d, "mask", "0.png"): os.path.join(d, "mask13", "0.png")} if face else None
        np.random.seed(1000 + c)
        with recorded(mod, files, alias) as rec:
            item = ds[index]
        pairs.append((item, rec["calls"][0]))
    return pairs, input_checksum(d, files), ds, files


def class_map_of(kind, call):
    from lib.utils.if_nerf import if_nerf_data_utils as du
    H, W = call["img"].shape[:2]
    bm = du.get_bound_2d_mask(call["bounds"], call["K"], np.concatenate([call["R"], call["T"]], axis=1), H, W)
    return (train_item.class_map_h36m if kind == "mv" else train_item.class_map_snapshot)(call["msk"], bm)


def make_golden(kind, cases, path):
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        pairs, sha, _, _ = reference_items(kind, cases, d)
    with tempfile.TemporaryDirectory() as d:
        (test_item, test_call), = reference_items(kind, ((TEST_INDEX, 1024, 0.5, 0.0, False),), d, "test")[0]
    arrays = {"input_sha256": np.frombuffer(sha.encode(), np.uint8), "cases": np.array(cases, dtype=np.float64)}
    # split 'test': every box-hit ray of the view, with its colour (if_nerf_data_utils.py:138-148 / :220-230)
    rgb, ray_o, ray_d, near, far, _, mask = test_call["out"]
    assert test_call["R"].dtype == np.float64 and 0 < mask.sum() < mask.size and len(rgb) == mask.sum()
    for k, x in (("img", test_call["img"]), ("K", test_call["K"]), ("R", test_call["R"]), ("T", test_call["T"]),
                 ("bounds", test_call["bounds"]), ("rgb", rgb), ("ray_o", ray_o), ("ray_d", ray_d), ("near", near),
                 ("far", far), ("mask_at_box", mask)):
        arrays["test_" + k] = x
    print("%s split 'test': %d of %d pixels hit the box" % (kind, int(mask.sum()), mask.size))
    max_rounds = 0
    for c, ((index, nrays, rb, rf, face), (item, call)) in enumerate(zip(cases, pairs)):
        rgb, ray_o, ray_d, near, far, coord, mask = call["out"]
        cmap = class_map_of(kind, call)
        draws = np.concatenate(call["draws"]) if call["draws"] else np.zeros(0, np.int64)
        rounds = len(call["draws"]) // (3 if (cmap & train_item.FACE).any() else 2)
        mine = sample_numpy(call["img"], cmap, call["K"], call["R"], call["T"], call["bounds"], nrays, rb, rf, draws)
        for a, b in zip(mine[:6], (rgb, ray_o, ray_d, near, far, coord)):
            assert a.dtype == b.dtype and np.array_equal(a, b), "restatement differs (%s case %d)" % (kind, c)
        assert mine[6] == rounds and len(near) == nrays and mask.all()
        assert not face or (cmap & train_item.FACE).any()
        assert call["R"].dtype == np.float64 and call["T"].dtype == np.float64 and call["bounds"].dtype == np.float32
        max_rounds = max(max_rounds, rounds)
        for k, x in (("img", call["img"]), ("msk", call["msk"]), ("K", call["K"]), ("R", call["R"]), ("T", call["T"]),
                     ("bounds", call["bounds"]), ("class_map", cmap), ("draws", draws), ("rounds", np.array(rounds)),
                     ("rgb", rgb), ("ray_o", ray_o), ("ray_d", ray_d), ("near", near), ("far", far), ("coord", coord)):
            arrays["%s_%d" % (k, c)] = x
        print("%s case %d: %d x %d, N_rand %d, ratios %.1f / %.1f, face pixels %d, border %s, %d rounds" % (
            kind, c, cmap.shape[0], cmap.shape[1], nrays, rb, rf, int((cmap & train_item.FACE).astype(bool).sum()), bool((call["msk"] == 100).any()), rounds))
    assert max_rounds >= 2, "no case needed a second round"
    np.savez_compressed(path, **arrays)
    print("-> %s (%d KB)" % (path, os.path.getsize(path) // 1024))


def load_golden(path):
    z = np.load(path)
    cases = [(int(c[0]), int(c[1]), float(c[2]), float(c[3]), bool(c[4])) for c in z["cases"]]
    keys = ("img", "msk", "K", "R", "T", "bounds", "class_map", "draws", "rounds", "rgb", "ray_o", "ray_d", "near", "far",
            "coord")
    test_keys = ("img", "K", "R", "T", "bounds", "rgb", "ray_o", "ray_d", "near", "far", "mask_at_box")
    return {"input_sha256": bytes(z["input_sha256"]).decode(), "cases": cases,
            "items": [{k: z["%s_%d" % (k, c)] for k in keys} for c in range(len(cases))],
            "test": {k: z["test_" + k] for k in test_keys}}


if __name__ == "__main__":
    make_golden("mv", MV_CASES, GOLDEN_MV)
    make_golden("mono", MONO_CASES, GOLDEN_MONO)
