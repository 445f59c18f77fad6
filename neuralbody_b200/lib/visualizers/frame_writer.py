"""The implementation the drop-ins lib/visualizers/if_nerf_demo.py and if_nerf_perform.py share: upstream's per-view body
(the rays scattered into a float64 H x W x 3 image over the background, BGR, `* 255`, `mkdir -p`, cv2.imwrite) with the
image built on the GPU and written off the view loop.

visualize(output, batch) enqueues on the current stream, with no host synchronisation:
  1. nb_vis_frame (neuralbody_b200.vis_frame): the uint8 BGR frame cv2.imwrite makes of upstream's float64 image, and a
     status record with the mask's count;
  2. a non-blocking copy of the frame and the record into a pinned slot, and of frame_index / view_index (device values;
     host values are written into the slot directly);
  3. a CUDA event.
One writer thread (neuralbody_b200.png_writer) waits on the slot's event, checks the status, makes the directory and calls
cv2.imwrite.  The slots form a bounded ring: visualize() waits for a free one, so a slow disk holds the loop back instead of
growing memory.

Differences from upstream, all about when things happen:
  - a PNG may not be on disk yet when visualize() returns.  flush() waits for every queued view; an atexit handler does
    the same when the process exits normally, so the last views are written;
  - a mask_at_box whose size is not H * W raises upstream's reshape ValueError at once; a mask count that does not match
    the rays (upstream's "shape mismatch" ValueError) and a writer error are raised by the next visualize() or flush(),
    and the views queued after it are not written;
  - upstream ignores a False from cv2.imwrite; here it is an IOError, as in the evaluator drop-in;
  - upstream also scatters output['depth_map'] into an image it never uses; that step is not run.
The PNG files are upstream's byte for byte."""
import atexit
import os
import queue
import weakref

import torch

from neuralbody_b200 import capi, vis_frame
from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.evaluators.if_nerf import _colored
from neuralbody_b200.png_writer import PngWriter

SLOTS = 4


class Slot:
    """The pinned host side of one queued view: `out` (vis_frame.ViewFrame.out's layout), `idx` (frame_index,
    view_index) int64, `n` (the view's rays) and the event the writer waits on."""

    def __init__(self, H, W, pin=True):
        self.H, self.W = int(H), int(W)
        self.out = torch.empty(vis_frame.FRAME_OFFSET + self.H * self.W * 3, dtype=torch.uint8, pin_memory=pin)
        self.idx = torch.empty(2, dtype=torch.int64, pin_memory=pin)
        self.n = 0
        self.event = torch.cuda.Event() if pin else None


def _flush_at_exit(ref):
    vis = ref()
    if vis is not None:
        vis.flush()


class FrameVisualizer:
    """Upstream's Visualizer() / visualize(output, batch), plus flush().  Subclasses give the output directory and the file
    of a view."""

    def data_dir(self, exp_name):
        raise NotImplementedError

    def frame_path(self, exp_name, frame_index, view_index):
        raise NotImplementedError

    def __init__(self):
        cfg = get_active_cfg()
        print(_colored('the results are saved at {}'.format(self.data_dir(cfg.exp_name)), 'yellow'))
        self._writer = PngWriter(depth=SLOTS, name="vis-png-writer")
        self._view = None        # vis_frame.ViewFrame of the current view size
        self._free = None        # queue.Queue of the free Slots of that size
        # registered after torch's own exit handlers, so it runs before them: the last views reach the disk
        atexit.register(_flush_at_exit, weakref.ref(self))

    def flush(self):
        """Wait until every queued view's PNG is written; raise the first error of any of them."""
        self._writer.join()

    def _buffers(self, H, W, device):
        v = self._view
        if v is None or (v.H, v.W, v.device) != (H, W, device):
            self.flush()             # every slot is free again
            self._view = vis_frame.ViewFrame(H, W, device)
            self._free = queue.Queue()
            for _ in range(SLOTS):
                self._free.put(Slot(H, W))
        return self._view

    def visualize(self, output, batch):
        cfg = get_active_cfg()
        self._writer.check()
        rgb = output['rgb_map'][0].detach()
        mask = batch['mask_at_box'][0].detach()
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        if mask.numel() != H * W:
            raise ValueError("cannot reshape array of size %d into shape (%d,%d)" % (mask.numel(), H, W))
        indices = (batch['frame_index'], batch['view_index'])
        dev = rgb.device if rgb.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        rgb, mask = rgb.to(dev, non_blocking=True), mask.to(dev, non_blocking=True)
        view = self._buffers(H, W, dev)
        slot = self._free.get()      # back-pressure: waits while every slot is queued
        try:
            view.launch(rgb, mask, int(cfg.white_bkgd))
            slot.out.copy_(view.out, non_blocking=True)
            for k, v in enumerate(indices):
                slot.idx[k:k + 1].copy_(torch.as_tensor(v).reshape(-1)[:1], non_blocking=True)
            slot.n = int(rgb.shape[0])
            slot.event.record(torch.cuda.current_stream(dev))
        except BaseException:
            self._free.put(slot)
            raise
        self._enqueue(slot, cfg.exp_name)

    def _enqueue(self, slot, exp_name):
        """Queue the writer's job for a filled slot; the slot is free again once the job is done or skipped."""
        free = self._free

        def make():
            status, count = vis_frame.parse(slot.out.numpy())
            if status != capi.NB_VIS_OK:
                raise ValueError("shape mismatch: value array of shape (%d,3) could not be broadcast to indexing result "
                                 "of shape (%d,3)" % (slot.n, count))
            fi, vi = (int(v) for v in slot.idx.tolist())
            path = self.frame_path(exp_name, fi, vi)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            return path, slot.out.numpy()[vis_frame.FRAME_OFFSET:].reshape(slot.H, slot.W, 3)

        self._writer.submit(make, slot.event, lambda: free.put(slot))

