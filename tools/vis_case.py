"""The demo visualizers' frame cases and the rotate-SMPL dataset's items (TEST INFRASTRUCTURE ONLY), and the generator of
their goldens.

`case(name)` rebuilds a seeded view from integers alone (so every machine rebuilds the same float32 bits): colours k / 255
on ramps with a block of random values, plus the case's special values, and a mask of the case's shape.  `run_reference`
runs the UNMODIFIED reference visualizers (lib/visualizers/if_nerf_demo.py, if_nerf_perform.py) through
oracle/ref_harness.py, with matplotlib.pyplot and termcolor stubbed, and returns the PNG bytes they write.
`reference_rotate_items` runs the UNMODIFIED reference rotate_smpl_dataset's __getitem__ on tools.demo_case's synthetic
ZJU-MoCap-like tree (imageio, plyfile stubbed) and records what it hands render_utils.image_rays.

    python -m tools.vis_case

writes, overwriting them:
  - tests/golden/vis_frames.npz: per case the decoded uint8 frame of the reference's PNG and a checksum of the rebuilt
    inputs;
  - tests/golden/vis_rotate.npz: for views ROTATE_VIEWS, the item's keys (coord, out_sh, bounds, R, Th, latent_index,
    frame_index, view_index), the camera and box image_rays received and its rays, near, far and mask_at_box, with the
    sha256 of the synthetic inputs (demo_case.input_checksum reproduces it without the reference tree)."""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools import demo_case as DC  # noqa: E402
from tools import eval_case as EC  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "vis_frames.npz")
GOLDEN_ROTATE = os.path.join(ROOT, "tests", "golden", "vis_rotate.npz")
# name: (H, W, white_bkgd, mask kind, special values, seed)
CASES = {
    "zju512": (512, 512, 0, "ellipse", None, 1),          # ZJU-MoCap at ratio 0.5
    "snapshot1080": (1080, 1080, 0, "tall", None, 2),     # People-Snapshot's size
    "white": (96, 128, 1, "ellipse", None, 3),
    "border": (64, 80, 0, "border", None, 4),             # the mask touches the top, left and right edges
    "empty": (40, 48, 1, "empty", None, 5),               # n = 0: an all-background frame
    "saturate": (60, 70, 0, "ellipse", "saturate", 6),    # below 0, above 1, outside int32, inf, NaN
    "ties": (48, 64, 1, "ellipse", "ties", 7),            # products on and next to k + 0.5
}
ROTATE_VIEWS = (0, 17, 71, 143)
ROTATE_KEYS = ("coord", "out_sh", "bounds", "R", "Th", "latent_index", "frame_index", "view_index")


def special_values(kind):
    if kind == "saturate":
        return np.array([-0.3, -1e-3, 1.0001, 1.7, 1e10, -1e10, 3e7, np.inf, -np.inf, np.nan, 0.0, 1.0], np.float32)
    # v * 255 in float64 is exact for a float32 v, and lands on k + 0.5 only for v = m / 2 (m odd); next to every tie
    # k + 0.5 of [0, 255) lie the float32 values nearest (2k + 1) / 510 and their neighbours
    near = np.array([(2 * k + 1) / 510.0 for k in range(255)], np.float32)
    return np.concatenate([np.array([0.5, 1.5, -0.5, 2.5, -1.5], np.float32), near,
                           np.nextafter(near, np.float32(np.inf)), np.nextafter(near, np.float32(-np.inf))])


def case(name):
    """-> rgb_map (n,3) float32, mask_at_box (H*W) bool, and the case's (H, W, white_bkgd)."""
    H, W, white, kind, special, seed = CASES[name]
    yy, xx = np.mgrid[0:H, 0:W].astype(np.int64)
    c = np.arange(3, dtype=np.int64)
    k = (3 * xx[..., None] + 5 * yy[..., None] + 40 * c + 17 * seed) % 256
    img = k.astype(np.float32) / np.float32(255)
    rng = np.random.RandomState(seed)
    bh, bw = min(24, H // 3), min(24, W // 3)
    y0, x0 = H // 2 - bh // 2, W // 2 - bw // 2
    img[y0:y0 + bh, x0:x0 + bw] = rng.rand(bh, bw, 3).astype(np.float32)
    mask = np.zeros((H, W), bool) if kind == "empty" else EC.mask_of(kind, H, W)
    rgb = np.ascontiguousarray(img[mask])
    if special is not None:
        vals = special_values(special)
        flat = rgb.reshape(-1)
        flat[:] = np.resize(vals, flat.size)
    return rgb, mask.reshape(-1), (H, W, white)


def checksum(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def random_view(H, W, seed):
    """A random view with an ellipse mask, values in [-0.1, 1.1) and a few NaN (the GPU tests' random cases)."""
    rng = np.random.RandomState(seed)
    cy, cx = rng.uniform(0.3, 0.7) * H, rng.uniform(0.3, 0.7) * W
    yy, xx = np.mgrid[0:H, 0:W]
    mask = ((xx - cx) / (rng.uniform(0.15, 0.45) * W)) ** 2 + ((yy - cy) / (rng.uniform(0.2, 0.45) * H)) ** 2 < 1
    n = int(mask.sum())
    rgb = (rng.rand(n, 3) * 1.2 - 0.1).astype(np.float32)
    rgb[rng.rand(n, 3) < 1e-3] = np.nan
    return rgb, mask.reshape(-1)


# ----------------------------------------------------------------------------- the unmodified reference visualizers
def reference_visualizers():
    """The reference's lib/visualizers/if_nerf_demo.py and if_nerf_perform.py modules and its cfg, loaded through
    oracle/ref_harness.py with a bare matplotlib.pyplot and a pass-through termcolor."""
    import importlib
    from oracle import ref_harness
    cfg = ref_harness.load_reference()[0]
    if "matplotlib" not in sys.modules:
        mpl, plt = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, plt
    if "termcolor" not in sys.modules:
        tc = types.ModuleType("termcolor")
        tc.colored = lambda text, *a, **k: text
        sys.modules["termcolor"] = tc
    if ref_harness.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_harness.REFERENCE_ROOT)
    mods = {k: importlib.import_module("lib.visualizers.if_nerf_" + k) for k in ("demo", "perform")}
    return mods, cfg


def reference_png(kind, rgb, mask, H, W, white, frame_index=3, view_index=11, exp_name="vis_case"):
    """The reference visualizer `kind` ('demo' or 'perform') on one view, in a temporary working directory -> the bytes of
    the PNG it writes."""
    import torch
    mods, cfg = reference_visualizers()
    old = os.getcwd()
    with tempfile.TemporaryDirectory() as d:
        os.chdir(d)
        try:
            cfg.H, cfg.W, cfg.ratio, cfg.white_bkgd, cfg.exp_name = H, W, 1.0, bool(white), exp_name
            vis = mods[kind].Visualizer()
            out = {"rgb_map": torch.from_numpy(rgb)[None], "depth_map": torch.zeros((1, rgb.shape[0]))}
            batch = {"mask_at_box": torch.from_numpy(mask)[None], "frame_index": torch.tensor([frame_index]),
                     "view_index": torch.tensor([view_index])}
            vis.visualize(out, batch)
            path = reference_path(kind, exp_name, frame_index, view_index)
            with open(path, "rb") as f:
                return f.read()
        finally:
            os.chdir(old)


def reference_path(kind, exp_name, frame_index, view_index):
    """Where upstream's visualizer `kind` writes a view (relative to the working directory)."""
    if kind == "demo":
        return os.path.join('data/render/{}/frame_{:04d}'.format(exp_name, frame_index), '{:04d}.png'.format(view_index))
    return os.path.join('data/perform/{}/0'.format(exp_name), 'frame{:04d}_view{:04d}.png'.format(frame_index, view_index))


def load_golden():
    z = np.load(GOLDEN)
    return {name: {k: z[name + "_" + k] for k in ("frame", "sha256")} for name in CASES}


# ----------------------------------------------------------------------------- the rotate-SMPL dataset
def rotate_setup():
    """The reference's cfg set for demo_case's synthetic tree, as its demo goldens set it."""
    cfg = DC._reference_setup()
    if "PIL" not in sys.modules:
        try:
            import PIL  # noqa: F401
        except ImportError:
            pil = types.ModuleType("PIL")
            pil.Image = object
            sys.modules["PIL"] = pil
    return cfg


def reference_rotate_items(views, d):
    """The UNMODIFIED reference rotate_smpl_dataset on demo_case's synthetic tree in `d` -> ([(item, image_rays call)],
    input sha256, dataset, module)."""
    rotate_setup()
    from lib.datasets.light_stage import rotate_smpl_dataset as mod
    masks = DC.write_mv_root(d)
    ds = mod.Dataset(d, "synthetic", os.path.join(d, "annots.npy"), "test")
    return DC._run_items(mod, ds, masks, views), DC.input_checksum(d, masks), ds, mod


def load_rotate_golden():
    z = np.load(GOLDEN_ROTATE)
    views = [int(v) for v in z["views"]]
    out = {"H": int(z["H"]), "W": int(z["W"]), "input_sha256": bytes(z["input_sha256"]).decode(), "views": {}}
    keys = ("RT", "K", "can_bounds", "ray_o", "ray_d", "near", "far", "mask_at_box") + ROTATE_KEYS
    for v in views:
        out["views"][v] = {k: z["%s_%d" % (k, v)] for k in keys}
    return out


def make_rotate_golden(path=GOLDEN_ROTATE):
    with tempfile.TemporaryDirectory() as d:
        pairs, sha, _, _ = reference_rotate_items(ROTATE_VIEWS, d)
    H, W = int(DC.RAW_HW[0] * DC.RATIO), int(DC.RAW_HW[1] * DC.RATIO)
    arrays = {"input_sha256": np.frombuffer(sha.encode(), np.uint8), "H": np.array(H), "W": np.array(W),
              "views": np.array(ROTATE_VIEWS)}
    for v, (item, call) in zip(ROTATE_VIEWS, pairs):
        ray_o, ray_d, near, far, _, _, mask = call["out"]
        mine = DC.image_rays_numpy(call["RT"], call["K"], call["bounds"], H, W)
        assert all(np.array_equal(a, b) for a, b in zip((ray_o, ray_d, near, far, mask), mine)), "restatement differs"
        assert 0 < mask.sum() < mask.size
        for k, x in (("RT", call["RT"]), ("K", call["K"]), ("can_bounds", call["bounds"]), ("ray_o", ray_o),
                     ("ray_d", ray_d), ("near", near), ("far", far), ("mask_at_box", mask)):
            arrays["%s_%d" % (k, v)] = x
        for k in ROTATE_KEYS:
            arrays["%s_%d" % (k, v)] = np.asarray(item[k])
    np.savez_compressed(path, **arrays)
    print("rotate: views %s, n = %s -> %s (%d KB)" % (ROTATE_VIEWS, [int(arrays["mask_at_box_%d" % v].sum()) for v in ROTATE_VIEWS],
                                                     path, os.path.getsize(path) // 1024))


def main():
    import cv2
    arrays = {}
    for name in CASES:
        rgb, mask, (H, W, white) = case(name)
        png = reference_png("demo", rgb, mask, H, W, white)
        if name in ("white", "border", "saturate"):
            assert reference_png("perform", rgb, mask, H, W, white) == png, name
        frame = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
        assert frame.shape == (H, W, 3) and frame.dtype == np.uint8
        arrays[name + "_frame"] = frame
        arrays[name + "_sha256"] = np.frombuffer(checksum(rgb, mask).encode(), np.uint8)
        print(name, (H, W, white), "n =", rgb.shape[0])
    np.savez_compressed(GOLDEN, **arrays)
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")
    make_rotate_golden()


if __name__ == "__main__":
    main()
