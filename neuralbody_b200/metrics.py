"""The evaluator's per-view metrics on the device (nb_eval_image): the scatter of a view's rays into its image, the MSE and
PSNR, the crop box, scikit-image 0.14.2's SSIM over the crop and the crops as uint8 BGR, as upstream's
lib/evaluators/if_nerf.py computes them on the host (oracle/eval_metrics.py restates them).  lib/evaluators/if_nerf.py
(this package's drop-in) reads the results back once per view."""
import ctypes as C

import numpy as np
import torch

from . import capi

RESULT_BYTES = C.sizeof(capi.nb_eval_image_result)
_CROP_OFFSET = 256          # the crops follow the result record, 256-byte aligned


class ViewEval:
    """Device buffers of nb_eval_image for one view size on one device, reused by every call: the workspace and one
    output buffer [result record | pred crop | gt crop], so that a single copy brings all of it back."""

    def __init__(self, H, W, device):
        lib = capi.load()
        self.H, self.W, self.device = int(H), int(W), torch.device(device)
        ws = lib.nb_eval_image_workspace_bytes(self.H, self.W, 0)
        if ws == 0:
            raise ValueError("H and W must be >= 1 with H*W < 2^31 (got %d x %d)" % (self.H, self.W))
        self.crop_bytes = self.H * self.W * 3
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=self.device)
        self.out = torch.empty(_CROP_OFFSET + 2 * self.crop_bytes, dtype=torch.uint8, device=self.device)
        self.result = self.out[:RESULT_BYTES]
        self.box = self.out[8:24].view(torch.int32)
        self.crop_pred = self.out[_CROP_OFFSET:_CROP_OFFSET + self.crop_bytes]
        self.crop_gt = self.out[_CROP_OFFSET + self.crop_bytes:]

    def launch(self, rgb_pred, rgb_gt, mask_at_box, white_bkgd=False, eval_whole_img=False):
        """Enqueue nb_eval_image on the current stream: rgb_pred, rgb_gt (n,3) float32 and mask_at_box (H*W) bool or
        uint8 (nonzero = set), all on this object's device.  Nothing synchronises with the host; the outputs are
        `result` (the nb_eval_image_result record's bytes), `box` (x, y, w, h int32) and `crop_pred` / `crop_gt`, whose
        first w*h*3 bytes are the crops (row-major, BGR)."""
        lib = capi.load()
        for name, t in (("rgb_pred", rgb_pred), ("rgb_gt", rgb_gt), ("mask_at_box", mask_at_box)):
            if not torch.is_tensor(t) or t.device != self.device:
                raise ValueError("%s must be a tensor on %s (got %s)" % (
                    name, self.device, t.device if torch.is_tensor(t) else type(t).__name__))
        if rgb_pred.dim() != 2 or rgb_pred.shape[1] != 3 or rgb_pred.shape != rgb_gt.shape or \
                rgb_pred.dtype != torch.float32 or rgb_gt.dtype != torch.float32:
            raise ValueError("rgb_pred and rgb_gt must both be (n,3) float32 (got %s %s, %s %s)"
                             % (tuple(rgb_pred.shape), rgb_pred.dtype, tuple(rgb_gt.shape), rgb_gt.dtype))
        if mask_at_box.numel() != self.H * self.W or mask_at_box.dtype not in (torch.bool, torch.uint8):
            raise ValueError("mask_at_box must hold H*W = %d bool or uint8 values (got %s %s)"
                             % (self.H * self.W, tuple(mask_at_box.shape), mask_at_box.dtype))
        rgb_pred, rgb_gt = rgb_pred.detach().contiguous(), rgb_gt.detach().contiguous()
        mask = mask_at_box.detach().reshape(-1).contiguous().view(torch.uint8)
        a = capi.nb_eval_image_args()
        a.n, a.H, a.W = int(rgb_pred.shape[0]), self.H, self.W
        a.white_bkgd, a.eval_whole_img = int(bool(white_bkgd)), int(bool(eval_whole_img))
        a.rgb_pred, a.rgb_gt, a.mask_at_box = rgb_pred.data_ptr(), rgb_gt.data_ptr(), mask.data_ptr()
        a.workspace, a.workspace_bytes = self.workspace.data_ptr(), self.workspace.numel()
        a.result, a.crop_pred, a.crop_gt = self.result.data_ptr(), self.crop_pred.data_ptr(), self.crop_gt.data_ptr()
        with torch.cuda.device(self.device):
            capi.check(lib.nb_eval_image(C.byref(a), C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                       "nb_eval_image")
        return self


def parse(out_host):
    """The host copy of ViewEval.out (a uint8 numpy array or tensor) -> dict: status, count, box (x, y, w, h), sq_sum,
    mse, psnr, ssim, ssim_channel, and crop_pred / crop_gt as (h, w, 3) uint8 BGR arrays (copies)."""
    buf = np.asarray(out_host)
    r = capi.nb_eval_image_result.from_buffer_copy(buf[:RESULT_BYTES].tobytes())
    x, y, w, h = (int(v) for v in r.box)
    n = w * h * 3 if r.status != capi.NB_EVAL_COUNT else 0
    crop_bytes = (buf.size - _CROP_OFFSET) // 2
    res = {"status": int(r.status), "count": int(r.count), "box": (x, y, w, h), "sq_sum": float(r.sq_sum),
           "mse": float(r.mse), "psnr": float(r.psnr), "ssim": float(r.ssim), "ssim_channel": tuple(r.ssim_channel)}
    if r.status == capi.NB_EVAL_OK:
        res["crop_pred"] = np.array(buf[_CROP_OFFSET:_CROP_OFFSET + n]).reshape(h, w, 3)
        res["crop_gt"] = np.array(buf[_CROP_OFFSET + crop_bytes:_CROP_OFFSET + crop_bytes + n]).reshape(h, w, 3)
    return res


def eval_image(rgb_pred, rgb_gt, mask_at_box, H, W, white_bkgd=False, eval_whole_img=False):
    """One view, with buffers of its own: -> the ViewEval whose device tensors (`result`, `box`, `crop_pred`, `crop_gt`)
    hold the outputs once the current stream reaches them.  `parse(v.out.cpu().numpy())` reads them."""
    return ViewEval(H, W, rgb_pred.device).launch(rgb_pred, rgb_gt, mask_at_box, white_bkgd, eval_whole_img)
