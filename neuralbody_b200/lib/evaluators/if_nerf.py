"""Drop-in for the reference's lib/evaluators/if_nerf.py (selected by `evaluator_module` / `evaluator_path`, as upstream's
make_evaluator loads it): the same `Evaluator()` with `evaluate(output, batch)` and `summarize()`, the same metrics, PNGs
and metrics.npy, with the per-view work on the GPU (neuralbody_b200.metrics, nb_eval_image):

  - the scatter of the view's rays into the H x W images, the MSE and PSNR, the crop box (cv2.boundingRect of
    mask_at_box), scikit-image 0.14.2's compare_ssim(multichannel=True) over the crop in float64, and the crops as the
    uint8 BGR bytes cv2.imwrite makes of upstream's float64 images, in six launches;
  - one host synchronisation per view, which brings back the result record, the crop bytes and the frame / view
    indices into pinned memory;
  - the two PNGs are encoded and written by one background thread (cv2.imwrite releases the GIL), so the next view
    renders meanwhile; a writer error is raised at the next evaluate() or at summarize().

Precision: the box and the PNG bytes are upstream's exactly; SSIM is upstream's float64 up to summation order (within
1e-12); the MSE is the float64 sum of upstream's float32 terms (eval_whole_img: of its float64 terms), so it is within a
few float32 ulps of numpy's float32 pairwise mean; PSNR is -10 log10 of that in float64.  summarize() returns the means as
a dict (upstream returns None, which Trainer.val cannot use)."""
import os

import numpy as np
import torch

from neuralbody_b200 import capi, metrics
from neuralbody_b200.png_writer import PngWriter
from neuralbody_b200.lib.config import get_active_cfg


def _colored(text, color):
    try:
        from termcolor import colored
    except ImportError:
        return text
    return colored(text, color)


class Evaluator:
    def __init__(self):
        self.mse = []
        self.psnr = []
        self.ssim = []
        self._view = None        # metrics.ViewEval of the current view size
        self._host = None        # its pinned readback buffer
        self._index = None       # pinned (2,) int64: frame_index, cam_ind
        self._writer = PngWriter(name="if_nerf-png-writer")

    def _buffers(self, H, W, device):
        v = self._view
        if v is None or (v.H, v.W, v.device) != (H, W, device):
            self._view = metrics.ViewEval(H, W, device)
            self._host = torch.empty(self._view.out.numel(), dtype=torch.uint8, pin_memory=True)
            self._index = torch.empty(2, dtype=torch.int64, pin_memory=True)
        return self._view

    def evaluate(self, output, batch):
        cfg = get_active_cfg()
        self._writer.check()
        frame_index, view_index = batch['frame_index'], batch['cam_ind']    # KeyError without them, as upstream
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        white_bkgd, whole = int(cfg.white_bkgd), bool(cfg.get('eval_whole_img', False))
        pred = output['rgb_map'][0]
        dev = pred.device if pred.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        pred = pred.detach().to(dev, non_blocking=True)
        gt = batch['rgb'][0].detach().to(dev, non_blocking=True)
        mask = batch['mask_at_box'][0].detach().to(dev, non_blocking=True)
        if mask.numel() != H * W:
            raise ValueError("cannot reshape array of size %d into shape (%d,%d)" % (mask.numel(), H, W))
        view = self._buffers(H, W, dev)
        view.launch(pred, gt, mask, white_bkgd, whole)
        self._host.copy_(view.out, non_blocking=True)
        idx = torch.stack([torch.as_tensor(frame_index).reshape(()).to(dev, torch.int64),
                           torch.as_tensor(view_index).reshape(()).to(dev, torch.int64)])
        self._index.copy_(idx, non_blocking=True)
        torch.cuda.current_stream(dev).synchronize()           # the view's one host synchronisation
        res = metrics.parse(self._host.numpy())
        if res["status"] == capi.NB_EVAL_COUNT:
            raise ValueError("shape mismatch: value array of shape (%d,3) could not be broadcast to indexing result of "
                             "shape (%d,3)" % (pred.shape[0], res["count"]))
        self.mse.append(np.float64(res["mse"]) if whole else np.float32(res["mse"]))
        self.psnr.append(np.float64(res["psnr"]))
        if res["status"] == capi.NB_EVAL_SMALL:
            raise ValueError("win_size exceeds image extent.  If the input is a multichannel (color) image, set "
                             "multichannel=True.")
        result_dir = os.path.join(cfg.result_dir, 'comparison')
        os.makedirs(result_dir, exist_ok=True)
        fi, vi = (int(v) for v in self._index.tolist())
        self._writer.put('{}/frame{:04d}_view{:04d}.png'.format(result_dir, fi, vi), res["crop_pred"])
        self._writer.put('{}/frame{:04d}_view{:04d}_gt.png'.format(result_dir, fi, vi), res["crop_gt"])
        self.ssim.append(np.float64(res["ssim"]))

    def summarize(self):
        cfg = get_active_cfg()
        self._writer.join()
        result_dir = cfg.result_dir
        print(_colored('the results are saved at {}'.format(result_dir), 'yellow'))
        result_path = os.path.join(cfg.result_dir, 'metrics.npy')
        os.makedirs(os.path.dirname(result_path) or '.', exist_ok=True)
        metrics_ = {'mse': self.mse, 'psnr': self.psnr, 'ssim': self.ssim}
        np.save(result_path, metrics_)
        means = {'mse': np.mean(self.mse), 'psnr': np.mean(self.psnr), 'ssim': np.mean(self.ssim)}
        print('mse: {}'.format(means['mse']))
        print('psnr: {}'.format(means['psnr']))
        print('ssim: {}'.format(means['ssim']))
        self.mse = []
        self.psnr = []
        self.ssim = []
        return means
