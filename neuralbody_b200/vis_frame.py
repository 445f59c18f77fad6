"""The demo visualizers' frame on the device (nb_vis_frame): the uint8 BGR image cv2.imwrite stores for upstream's
lib/visualizers/if_nerf_demo.py / if_nerf_perform.py float64 image of a view's rays (oracle/vis_frames.py restates it).
lib/visualizers/frame_writer.py (this package's drop-ins) copies it back and writes it off the view loop."""
import ctypes as C

import numpy as np
import torch

from . import capi

FRAME_OFFSET = 256          # the frame follows the status record, 256-byte aligned


class ViewFrame:
    """Device buffers of nb_vis_frame for one view size on one device, reused by every call: the workspace and one output
    buffer `out` = [nb_vis_frame_result | pad | frame (H,W,3)], so that a single copy brings both back."""

    def __init__(self, H, W, device):
        lib = capi.load()
        self.H, self.W, self.device = int(H), int(W), torch.device(device)
        ws = lib.nb_vis_frame_workspace_bytes(self.H, self.W)
        if ws == 0:
            raise ValueError("H and W must be >= 1 with H*W < 2^31 (got %d x %d)" % (self.H, self.W))
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=self.device)
        self.out = torch.empty(FRAME_OFFSET + self.H * self.W * 3, dtype=torch.uint8, device=self.device)
        self.result = self.out[:C.sizeof(capi.nb_vis_frame_result)]
        self.frame = self.out[FRAME_OFFSET:].view(self.H, self.W, 3)

    def launch(self, rgb_map, mask_at_box, white_bkgd=False):
        """Enqueue nb_vis_frame on the current stream: rgb_map (n,3) float32 and mask_at_box (H*W) bool or uint8
        (nonzero = set), on this object's device.  Nothing synchronises with the host; the outputs are `result` (the
        status record's bytes) and `frame`."""
        lib = capi.load()
        for name, t in (("rgb_map", rgb_map), ("mask_at_box", mask_at_box)):
            if not torch.is_tensor(t) or t.device != self.device:
                raise ValueError("%s must be a tensor on %s (got %s)" % (
                    name, self.device, t.device if torch.is_tensor(t) else type(t).__name__))
        if rgb_map.dim() != 2 or rgb_map.shape[1] != 3 or rgb_map.dtype != torch.float32:
            raise ValueError("rgb_map must be (n,3) float32 (got %s %s)" % (tuple(rgb_map.shape), rgb_map.dtype))
        if mask_at_box.numel() != self.H * self.W or mask_at_box.dtype not in (torch.bool, torch.uint8):
            raise ValueError("mask_at_box must hold H*W = %d bool or uint8 values (got %s %s)"
                             % (self.H * self.W, tuple(mask_at_box.shape), mask_at_box.dtype))
        rgb_map = rgb_map.detach().contiguous()
        mask = mask_at_box.detach().reshape(-1).contiguous().view(torch.uint8)
        a = capi.nb_vis_frame_args()
        a.n, a.H, a.W, a.white_bkgd = int(rgb_map.shape[0]), self.H, self.W, int(bool(white_bkgd))
        a.rgb_map, a.mask_at_box = rgb_map.data_ptr(), mask.data_ptr()
        a.workspace, a.workspace_bytes = self.workspace.data_ptr(), self.workspace.numel()
        a.result, a.frame = self.result.data_ptr(), self.frame.data_ptr()
        with torch.cuda.device(self.device):
            capi.check(lib.nb_vis_frame(C.byref(a), C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                       "nb_vis_frame")
        return self


def parse(out_host):
    """The host copy of ViewFrame.out (uint8 numpy array or tensor) -> (status, count)."""
    r = capi.nb_vis_frame_result.from_buffer_copy(np.asarray(out_host)[:C.sizeof(capi.nb_vis_frame_result)].tobytes())
    return int(r.status), int(r.count)


def vis_frame(rgb_map, mask_at_box, H, W, white_bkgd=False):
    """One view, with buffers of its own: -> the ViewFrame whose `result` and `frame` hold the outputs once the current
    stream reaches them."""
    return ViewFrame(H, W, rgb_map.device).launch(rgb_map, mask_at_box, white_bkgd)
