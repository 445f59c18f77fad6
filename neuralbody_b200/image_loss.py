"""The image losses of upstream's training wrapper on the device (nb_image_loss_fwd / nb_image_loss_bwd):
img_loss = torch.mean((rgb_map[mask] - rgb[mask]) ** 2) and img_loss0 = torch.mean((rgb0 - rgb) ** 2)
(lib/train/trainers/if_nerf_clight.py:24-32), without the boolean-mask index, whose nonzero makes the host wait for the
forward pass before it can queue the backward.  lib/train/trainers/if_nerf_clight.py (this package's drop-in) calls
`image_mse`.  The loss is summed in float64 in a fixed order (the same bits on every run); its gradient is the cotangent
autograd computes on the GPU for upstream's expression, bit for bit."""
import ctypes as C

import torch

from . import capi

_workspaces = {}


def _workspace(dev, stream):
    """The forward's partials and ticket for one (device, stream): zeroed once here, left zeroed by every forward, and only
    ever read in the stream's order."""
    key = (dev, stream)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(capi.load().nb_image_loss_workspace_bytes(), dtype=torch.uint8, device=dev)
        _workspaces[key] = ws
    return ws


def _args(pred, gt, mask):
    a = capi.nb_image_loss_args()
    a.rays = int(pred.numel() // 3)
    a.pred, a.gt = pred.data_ptr(), gt.data_ptr()
    a.mask = mask.data_ptr() if mask is not None else None
    return a


class _ImageMSE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, gt, mask):
        dev = pred.device
        pred_c, gt_c = pred.detach().contiguous(), gt.detach().contiguous()
        mask_c = None if mask is None else mask.detach().reshape(-1).contiguous().view(torch.uint8)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        count = torch.empty((), dtype=torch.int64, device=dev)
        a = _args(pred_c, gt_c, mask_c)
        a.loss, a.count = loss.data_ptr(), count.data_ptr()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            ws = _workspace(dev, stream)
            a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
            capi.check(capi.load().nb_image_loss_fwd(C.byref(a), C.c_void_p(stream)), "nb_image_loss_fwd")
        ctx.save_for_backward(pred_c, gt_c, count, *(() if mask_c is None else (mask_c,)))
        ctx.mark_non_differentiable(count)
        ctx.set_materialize_grads(False)
        return loss, count

    @staticmethod
    def backward(ctx, d_loss, _d_count):
        if d_loss is None or not ctx.needs_input_grad[0]:
            return None, None, None
        pred, gt, count, *mask = ctx.saved_tensors
        mask = mask[0] if mask else None
        dev = pred.device
        d_loss = d_loss.to(device=dev, dtype=torch.float32).contiguous()
        d_pred = torch.empty_like(pred)
        a = _args(pred, gt, mask)
        a.count = count.data_ptr()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(capi.load().nb_image_loss_bwd(C.byref(a), d_loss.data_ptr(), d_pred.data_ptr(), C.c_void_p(stream)),
                       "nb_image_loss_bwd")
        return d_pred, None, None


def _check(pred, gt, mask):
    for name, t in (("pred", pred), ("gt", gt)):
        if not torch.is_tensor(t) or t.device.type != "cuda" or t.dtype != torch.float32:
            raise ValueError("%s must be a float32 CUDA tensor (got %s)" % (
                name, "%s %s" % (t.dtype, t.device) if torch.is_tensor(t) else type(t).__name__))
    if pred.device != gt.device or pred.shape != gt.shape or pred.dim() < 1 or pred.shape[-1] != 3:
        raise ValueError("pred and gt must both be (..., 3) on one device (got %s on %s, %s on %s)"
                         % (tuple(pred.shape), pred.device, tuple(gt.shape), gt.device))
    if pred.numel() >= (1 << 31):
        raise ValueError("at most 2^31 - 1 elements (got %d)" % pred.numel())
    if gt.requires_grad and torch.is_grad_enabled():
        raise ValueError("gt must not require grad: the kernel differentiates pred only (upstream's target is a constant)")
    if mask is not None:
        if not torch.is_tensor(mask) or mask.dtype not in (torch.bool, torch.uint8) or mask.device != pred.device:
            raise ValueError("mask must be a bool or uint8 tensor on %s (got %s)" % (
                pred.device, "%s %s" % (mask.dtype, mask.device) if torch.is_tensor(mask) else type(mask).__name__))
        if tuple(mask.shape) != tuple(pred.shape[:-1]):
            # upstream's rgb_map[mask] raises IndexError here too
            raise IndexError("the mask's shape %s does not match the rays' %s" % (tuple(mask.shape), tuple(pred.shape[:-1])))


def image_mse(pred, gt, mask=None, with_count=False):
    """torch.mean((pred[mask] - gt[mask]) ** 2), or torch.mean((pred - gt) ** 2) without a mask, as a 0-dim float32 tensor
    on pred's device, with no host synchronisation.  pred, gt: (..., 3) float32 CUDA tensors of one shape (pred may require
    grad; gt's gradient is not computed); mask: bool or uint8 (nonzero = set) of pred.shape[:-1].  No set ray gives NaN,
    as upstream.  with_count: also return the number of elements averaged (0-dim int64 on the device)."""
    _check(pred, gt, mask)
    loss, count = _ImageMSE.apply(pred, gt, mask)
    return (loss, count) if with_count else loss
