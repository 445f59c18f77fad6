"""The evaluator without a GPU: the SSIM restatement against its definition, the oracle evaluator against the unmodified
reference evaluator (metrics and PNG bytes), the goldens, nb_eval_image's argument validation and the drop-in's loading
through the evaluator_module / evaluator_path factory."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import eval_metrics as O
from oracle import ref_harness
from tools import eval_case as EC


@pytest.fixture(scope="module", autouse=True)
def _unload_reference():
    """The reference evaluator imports the reference's `lib` package, which makes get_active_cfg() answer with the
    reference's cfg; take it out again after this module so later tests see this package's cfg."""
    import sys
    before = set(sys.modules)
    yield
    for name in set(sys.modules) - before:
        if name == "lib" or name.startswith("lib.") or name in ("skimage", "skimage.measure", "termcolor"):
            del sys.modules[name]
    ref_harness._loaded = None


# ----------------------------------------------------------------------------- the SSIM restatement
@pytest.mark.parametrize("shape", [(7, 7), (7, 19), (33, 12), (64, 64), (219, 399)])
def test_ssim_restatement_equals_the_definition(shape):
    rng = np.random.RandomState(shape[0] * 1000 + shape[1])
    X = rng.rand(*shape, 3)
    Y = np.clip(X + rng.normal(0, 0.1, X.shape), 0, 1)
    a, b = O.compare_ssim(X, Y, multichannel=True), O.ssim_bruteforce(X, Y)
    assert abs(a - b) <= 1e-13, (a, b)


def test_ssim_restatement_on_constant_and_equal_images():
    X = np.full((9, 11, 3), 0.25)
    Y = np.full((9, 11, 3), 0.75)
    assert abs(O.compare_ssim(X, Y, multichannel=True) - O.ssim_bruteforce(X, Y)) <= 1e-13
    Z = np.random.RandomState(0).rand(20, 30, 3)
    assert O.compare_ssim(Z, Z.copy(), multichannel=True) == 1.0
    with pytest.raises(ValueError):
        O.compare_ssim(np.zeros((6, 30, 3)), np.zeros((6, 30, 3)), multichannel=True)


def test_u8_conversion_and_box_are_opencvs():
    cv2 = pytest.importorskip("cv2")
    v = np.array([[[0.5, 1.5, -0.1], [1e10, np.inf, -np.inf], [np.nan, 1.0, 0.0], [2.5 / 255, 3.5 / 255, 0.3]]])
    img = v * 255
    ok, png = cv2.imencode(".png", img)
    assert ok and np.array_equal(cv2.imdecode(png, cv2.IMREAD_UNCHANGED), O.to_u8(img))
    for name in EC.CASES:
        _, _, mask, (H, W, _, _) = EC.case(name)
        m = mask.reshape(H, W)
        assert O.bounding_rect(m) == tuple(cv2.boundingRect(m.astype(np.uint8))), name
    assert O.bounding_rect(np.zeros((5, 5), bool)) == tuple(cv2.boundingRect(np.zeros((5, 5), np.uint8)))


# ----------------------------------------------------------------------------- the oracle against the reference
needs_reference = pytest.mark.skipif(not ref_harness.reference_available(), reason="needs the reference tree")


def _oracle_pngs(out, d):
    import cv2
    cv2.imwrite(os.path.join(d, "p.png"), out["crop_pred"])
    cv2.imwrite(os.path.join(d, "g.png"), out["crop_gt"])
    return open(os.path.join(d, "p.png"), "rb").read(), open(os.path.join(d, "g.png"), "rb").read()


def _same_metrics(out, ref):
    for k in ("mse", "psnr", "ssim"):
        assert type(out[k]) is type(ref[k]) and np.array_equal(out[k], ref[k], equal_nan=True), (k, out[k], ref[k])


@needs_reference
@pytest.mark.parametrize("name", sorted(EC.CASES))
def test_oracle_equals_the_reference_evaluator(name, tmp_path):
    pytest.importorskip("cv2")
    pred, gt, mask, (H, W, white, whole) = EC.case(name)
    ref = EC.run_reference(name)
    out = O.evaluate_view(pred, gt, mask, H, W, white, whole)
    _same_metrics(out, ref)
    assert _oracle_pngs(out, str(tmp_path)) == (ref["png_pred"], ref["png_gt"])
    # the upstream-path variant (cv2.boundingRect, PNGs from the float64 images) writes the same files
    up = O.evaluate_view(pred, gt, mask, H, W, white, whole, png_dir=str(tmp_path), frame_index=3, view_index=11)
    _same_metrics(up, ref)
    assert open(tmp_path / "frame0003_view0011.png", "rb").read() == ref["png_pred"]
    assert open(tmp_path / "frame0003_view0011_gt.png", "rb").read() == ref["png_gt"]


@needs_reference
def test_oracle_equals_the_reference_on_saturating_values(tmp_path):
    pytest.importorskip("cv2")
    mod, cfg = EC.reference_evaluator()
    pred, gt, mask = EC.random_view(40, 52, 5, special=True)
    ref = EC.run_reference_view(mod, cfg, pred, gt, mask, 40, 52, 0, 0)
    out = O.evaluate_view(pred, gt, mask, 40, 52)
    _same_metrics(out, ref)
    assert _oracle_pngs(out, str(tmp_path)) == (ref["png_pred"], ref["png_gt"])


@needs_reference
def test_reference_raises_where_the_oracle_does():
    mod, cfg = EC.reference_evaluator()
    pred, gt, mask, (H, W, _, _) = EC.case("small")
    for args in ((pred[:-1], gt[:-1], mask), ):
        with pytest.raises(ValueError):
            EC.run_reference_view(mod, cfg, *args, H, W, 0, 0)
        with pytest.raises(ValueError):
            O.evaluate_view(*args, H, W)
    m = np.zeros((H, W), bool)
    m[5:25, 10:16] = True                       # 6 pixels wide
    n = int(m.sum())
    for fn in (lambda: EC.run_reference_view(mod, cfg, pred[:n], gt[:n], m.reshape(-1), H, W, 0, 0),
               lambda: O.evaluate_view(pred[:n], gt[:n], m.reshape(-1), H, W)):
        with pytest.raises(ValueError, match="win_size"):
            fn()


# ----------------------------------------------------------------------------- the goldens
def test_goldens_load_and_match_the_oracle():
    g = EC.load_golden()
    assert set(g) == set(EC.CASES)
    for name, want in g.items():
        pred, gt, mask, (H, W, white, whole) = EC.case(name)
        assert EC.checksum(pred, gt, mask) == bytes(want["sha256"]).decode(), name
        out = O.evaluate_view(pred, gt, mask, H, W, white, whole)
        assert tuple(want["box"]) == out["box"], name
        assert np.array_equal(want["crop_pred"], out["crop_pred"]) and np.array_equal(want["crop_gt"], out["crop_gt"])
        for k in ("mse", "psnr", "ssim"):
            assert want[k] == out[k], (name, k)
    x, y, w, h = g["crop7"]["box"]
    assert w == 7 and g["border"]["box"][0] == 0 and g["border"]["box"][1] == 0
    assert os.path.getsize(EC.GOLDEN) < 1 << 20


# ----------------------------------------------------------------------------- the C ABI and the drop-in
def test_c_abi_validates_its_arguments(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_eval_image_workspace_bytes(0, 512, 0) == 0
    assert lib.nb_eval_image_workspace_bytes(512, 512, -1) == 0
    assert lib.nb_eval_image_workspace_bytes(65536, 65536, 0) == 0
    ws = lib.nb_eval_image_workspace_bytes(16, 16, 10) or 1 << 20    # the CUB size query needs a device

    def args(**kw):
        a = capi.nb_eval_image_args()
        a.n, a.H, a.W = 10, 16, 16
        a.rgb_pred = a.rgb_gt = a.mask_at_box = a.workspace = a.result = a.crop_pred = a.crop_gt = 256
        a.workspace_bytes = ws
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for kw in ({"mask_at_box": None}, {"rgb_pred": None}, {"result": None}, {"crop_gt": None}, {"workspace": None},
               {"H": 0}, {"n": -1}, {"white_bkgd": 2}, {"eval_whole_img": -1}, {"workspace_bytes": ws - 1}):
        assert lib.nb_eval_image(C.byref(args(**kw)), None) == -1, kw   # NB_ERR_BAD_ARG
        assert b"nb_eval_image" in lib.nb_last_error()
    assert C.sizeof(capi.nb_eval_image_result) == 80


def test_result_layout_matches_the_header(built_lib):
    import subprocess
    import tempfile
    from conftest import ROOT
    from neuralbody_b200 import capi
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "neuralbody_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
           'sizeof(nb_eval_image_result), sizeof(nb_eval_image_args), offsetof(nb_eval_image_result, box), '
           'offsetof(nb_eval_image_result, ssim_channel));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "p")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(capi.nb_eval_image_result), C.sizeof(capi.nb_eval_image_args),
                     capi.nb_eval_image_result.box.offset, capi.nb_eval_image_result.ssim_channel.offset]


def test_drop_in_loads_through_the_factory_with_upstreams_keys(tmp_path):
    """make_evaluator.py:5-9: imp.load_source(cfg.evaluator_module, cfg.evaluator_path).Evaluator(); the drop-in reads
    upstream's keys, and a missing cam_ind is upstream's KeyError (raised before anything runs on the device)."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.config.config import _defaults
    from neuralbody_b200.lib.networks.make_network import load_source
    d = _defaults()
    assert d.evaluator_module == cfg.evaluator_module == "neuralbody_b200.lib.evaluators.if_nerf"
    assert d.eval_whole_img is False and d.result_dir == "data/result"
    ev = load_source(cfg.evaluator_module, cfg.evaluator_path).Evaluator()
    assert ev.mse == [] and ev.psnr == [] and ev.ssim == []
    with pytest.raises(KeyError):
        ev.evaluate({"rgb_map": None}, {"frame_index": 0})
