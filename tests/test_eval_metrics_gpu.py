"""nb_eval_image and the evaluator drop-in on the GPU: the goldens made by the unmodified reference evaluator, the numpy
oracle (oracle/eval_metrics.py, pinned to the reference by test_eval_metrics_cpu) on random views, the exact cases, the
errors, and Renderer.render -> Evaluator.evaluate on a test-split view."""
import os

import numpy as np
import pytest
import torch

from oracle import eval_metrics as O
from tools import eval_case as EC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _restore_cfg():
    """The tests set cfg keys (sizes, result_dir, render options); later tests see the cfg as it was."""
    from neuralbody_b200.lib.config import cfg
    saved = cfg.clone()
    yield
    cfg.clear()
    cfg.update(saved)


def _gpu(pred, gt, mask, H, W, white=0, whole=0):
    from neuralbody_b200 import metrics
    v = metrics.eval_image(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), torch.from_numpy(mask).to(DEV),
                           H, W, white, whole)
    torch.cuda.synchronize()
    host = v.out.cpu().numpy()
    return metrics.parse(host), host


def _png(img):
    import cv2
    ok, buf = cv2.imencode(".png", img)
    assert ok
    return buf.tobytes()


def _check(got, want, label, mse_f64=None):
    assert got["status"] == 0, label
    assert got["box"] == tuple(int(v) for v in want["box"]), (label, got["box"], want["box"])
    for k in ("crop_pred", "crop_gt"):
        assert got[k].shape == want[k].shape and np.array_equal(got[k], want[k]), (label, k)
        if _has_cv2():
            assert _png(got[k]) == _png(want[k]), (label, k)
    assert abs(got["ssim"] - float(want["ssim"])) <= 1e-12, (label, got["ssim"], float(want["ssim"]))
    if mse_f64 is not None:
        assert abs(got["mse"] - mse_f64) <= 1e-12 * mse_f64, (label, got["mse"], mse_f64)
    assert abs(got["mse"] - float(want["mse"])) <= 4e-6 * float(want["mse"]), (label, got["mse"], float(want["mse"]))
    assert abs(got["psnr"] - float(want["psnr"])) <= 5e-5, (label, got["psnr"], float(want["psnr"]))
    print("%s: box %s, ssim %.3e, mse %.3e (rel), psnr %.3e dB from upstream" % (
        label, got["box"], abs(got["ssim"] - float(want["ssim"])), abs(got["mse"] / float(want["mse"]) - 1),
        abs(got["psnr"] - float(want["psnr"]))))


def _has_cv2():
    try:
        import cv2  # noqa: F401
        return True
    except ImportError:
        return False


@pytest.mark.parametrize("name", sorted(EC.CASES))
def test_goldens(name):
    """The reference evaluator's box, comparison images, SSIM, MSE and PSNR on every golden case."""
    want = EC.load_golden()[name]
    pred, gt, mask, (H, W, white, whole) = EC.case(name)
    assert EC.checksum(pred, gt, mask) == bytes(want["sha256"]).decode()
    got, _ = _gpu(pred, gt, mask, H, W, white, whole)
    _check(got, want, name, O.evaluate_view(pred, gt, mask, H, W, white, whole)["mse_f64"])


RANDOM = [(37, 41, 0, 0, 1), (128, 96, 1, 0, 2), (512, 512, 0, 0, 3), (1080, 700, 0, 0, 4), (200, 160, 1, 1, 5),
          (1080, 1080, 0, 1, 6)]


@pytest.mark.parametrize("case", RANDOM, ids=["%dx%d_w%d_whole%d" % c[:4] for c in RANDOM])
def test_random_views_equal_the_oracle(case):
    H, W, white, whole, seed = case
    pred, gt, mask = EC.random_view(H, W, seed)
    want = O.evaluate_view(pred, gt, mask, H, W, white, whole)
    got, _ = _gpu(pred, gt, mask, H, W, white, whole)
    _check(got, want, str(case), want["mse_f64"])


def test_saturating_values_give_opencvs_bytes():
    pred, gt, mask = EC.random_view(60, 70, 9, special=True)
    want = O.evaluate_view(pred, gt, mask, 60, 70)
    got, _ = _gpu(pred, gt, mask, 60, 70)
    assert got["box"] == want["box"]
    assert np.array_equal(got["crop_pred"], want["crop_pred"]) and np.array_equal(got["crop_gt"], want["crop_gt"])
    assert np.isnan(got["ssim"]) and np.isnan(want["ssim"])


def test_equal_images_and_two_runs():
    """pred == gt: SSIM exactly 1, MSE 0, PSNR +inf; and the same inputs give the same bytes twice."""
    pred, gt, mask = EC.random_view(300, 240, 11)
    got, _ = _gpu(pred, pred.copy(), mask, 300, 240)
    assert got["ssim"] == 1.0 and got["mse"] == 0.0 and got["psnr"] == np.inf
    assert all(c == 1.0 for c in got["ssim_channel"])
    a = _gpu(pred, gt, mask, 300, 240)[1]
    b = _gpu(pred, gt, mask, 300, 240)[1]
    n = 256 + 2 * 300 * 240 * 3
    assert np.array_equal(a[:80], b[:80]) and np.array_equal(a[256:n], b[256:n])


def test_statuses():
    from neuralbody_b200 import capi
    pred, gt, mask, (H, W, _, _) = EC.case("small")
    assert _gpu(pred[:-1], gt[:-1], mask, H, W)[0]["status"] == capi.NB_EVAL_COUNT
    m = np.zeros((H, W), bool)
    m[5:25, 10:16] = True
    n = int(m.sum())
    got = _gpu(pred[:n], gt[:n], m.reshape(-1), H, W)[0]
    assert got["status"] == capi.NB_EVAL_SMALL and got["box"] == (10, 5, 6, 20)
    assert np.isfinite(got["mse"])
    got = _gpu(pred[:0], gt[:0], np.zeros(H * W, bool), H, W, 1, 1)[0]     # empty mask, whole image: all background
    assert got["status"] == 0 and got["mse"] == 0.0 and got["ssim"] == 1.0


# ----------------------------------------------------------------------------- the drop-in
def _cfg(H, W, white, whole, result_dir):
    from neuralbody_b200.lib.config import cfg
    cfg.H, cfg.W, cfg.ratio = H, W, 1.0
    cfg.white_bkgd, cfg.eval_whole_img, cfg.result_dir = bool(white), bool(whole), str(result_dir)
    return cfg


def _evaluator():
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    return load_source(cfg.evaluator_module, cfg.evaluator_path).Evaluator()


def _view_batch(pred, gt, mask, frame, view, device=DEV):
    out = {"rgb_map": torch.from_numpy(pred)[None].to(device)}
    batch = {"rgb": torch.from_numpy(gt)[None].to(device), "mask_at_box": torch.from_numpy(mask)[None].to(device),
             "frame_index": torch.tensor([frame]).to(device), "cam_ind": torch.tensor([view]).to(device)}
    return out, batch


def test_evaluator_errors(tmp_path):
    pred, gt, mask, (H, W, _, _) = EC.case("small")
    _cfg(H, W, 0, 0, tmp_path)
    ev = _evaluator()
    with pytest.raises(ValueError, match="shape mismatch"):
        ev.evaluate(*_view_batch(pred[:-1], gt[:-1], mask, 0, 0))
    m = np.zeros((H, W), bool)
    m[5:25, 10:16] = True
    n = int(m.sum())
    with pytest.raises(ValueError, match="win_size"):
        ev.evaluate(*_view_batch(pred[:n], gt[:n], m.reshape(-1), 0, 0))
    out, batch = _view_batch(pred, gt, mask, 0, 0)
    del batch["cam_ind"]
    with pytest.raises(KeyError):
        ev.evaluate(out, batch)


def test_evaluator_writes_upstreams_files(tmp_path):
    """Views from device and host tensors: the PNGs are the reference's bytes (the goldens' images), metrics.npy has
    upstream's dict and element dtypes, and summarize() returns the means."""
    names = ("zju512", "holes", "whole")
    ev = _evaluator()
    got = {}
    for f, name in enumerate(names):
        pred, gt, mask, (H, W, white, whole) = EC.case(name)
        d = tmp_path / name
        _cfg(H, W, white, whole, d)
        ev.evaluate(*_view_batch(pred, gt, mask, f, 2 * f, DEV if f != 1 else torch.device("cpu")))
        got[name] = (d, f)
        means = ev.summarize()
        want = EC.load_golden()[name]
        m = np.load(d / "metrics.npy", allow_pickle=True).item()
        assert sorted(m) == ["mse", "psnr", "ssim"] and all(len(v) == 1 for v in m.values())
        assert type(m["mse"][0]) is (np.float64 if whole else np.float32)
        assert type(m["psnr"][0]) is np.float64 and type(m["ssim"][0]) is np.float64
        assert abs(m["ssim"][0] - want["ssim"]) <= 1e-12 and abs(m["psnr"][0] - want["psnr"]) <= 5e-5
        assert abs(float(m["mse"][0]) / float(want["mse"]) - 1) <= 4e-6
        assert means["ssim"] == m["ssim"][0] and means["psnr"] == m["psnr"][0]
        if _has_cv2():
            png = d / "comparison" / ("frame%04d_view%04d" % (f, 2 * f))
            assert open(str(png) + ".png", "rb").read() == _png(want["crop_pred"])
            assert open(str(png) + "_gt.png", "rb").read() == _png(want["crop_gt"])
    assert ev.mse == [] and ev.psnr == [] and ev.ssim == []


def test_render_then_evaluate_on_a_test_split_view(tmp_path):
    """A synth-313 test-split view (512 x 512, the image and camera in the batch): Renderer.render builds its rays, rgb and
    mask_at_box on the device, Evaluator.evaluate scores rgb_map; the oracle evaluator on the same rgb_map agrees."""
    from gpu_utils import make_net_and_renderer
    from neuralbody_b200.lib.config import cfg
    from tools.bench_eval import test_view
    scene, batch = test_view(512, DEV)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    _, ren = make_net_and_renderer(scene)
    with torch.no_grad():
        out = ren.render(batch)
    cfg.H, cfg.W, cfg.ratio, cfg.eval_whole_img, cfg.result_dir = 1024, 1024, 0.5, False, str(tmp_path)
    ev = _evaluator()
    ev.evaluate(out, batch)
    means = ev.summarize()
    pred, gt = out["rgb_map"][0].cpu().numpy(), batch["rgb"][0].cpu().numpy()
    mask = batch["mask_at_box"][0].cpu().numpy()
    want = O.evaluate_view(pred, gt, mask, 512, 512)
    assert abs(means["ssim"] - want["ssim"]) <= 1e-12
    assert abs(float(means["mse"]) / float(want["mse"]) - 1) <= 4e-6 and abs(means["psnr"] - want["psnr"]) <= 5e-5
    if _has_cv2():
        png = tmp_path / "comparison" / "frame0000_view0000"
        assert open(str(png) + ".png", "rb").read() == _png(want["crop_pred"])
        assert open(str(png) + "_gt.png", "rb").read() == _png(want["crop_gt"])
    print("render + evaluate: box %s, ssim %.6f" % (want["box"], means["ssim"]))
