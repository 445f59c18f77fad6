"""Drop-in for the reference's lib/visualizers/if_nerf_mesh.py (selected by `visualizer_module` / `visualizer_path`, as
upstream's make_visualizer loads it; `run.py --type visualize` with `vis_mesh True`): the same `Visualizer()` and
`visualize(output, batch)`, writing {cfg.result_dir}/mesh/{frame_index:04d}.ply, with the file written by a background
thread (neuralbody_b200.png_writer; call flush() to wait for the files).

visualize(output, batch) takes either kind of output['mesh'] the mesh renderer returns:
  - a neuralbody_b200.mcubes.DeviceMesh (`mesh_output: 'device'`): it enqueues nb_mesh_ply (DeviceMesh.pack), a
    non-blocking copy of the status record and PLY body into a pinned slot, a copy of frame_index (a device value; a host
    value is written into the slot directly) and a CUDA event.  Nothing synchronises with the host.  The writer thread
    waits on the event, checks the status and writes the header and the body;
  - a host mesh (trimesh.Trimesh or mcubes.Mesh, `mesh_output: 'host'`): the writer thread calls its export(path).
The slots form a ring of SLOTS: visualize() waits for a free one, so a slow disk holds the loop back instead of growing
memory.  A slot's pinned buffer is replaced only when a frame's body needs more bytes than it holds.

Differences from upstream, all about when things happen:
  - a PLY file may not be on disk yet when visualize() returns.  flush() waits for every queued frame; an atexit handler
    does the same when the process exits normally;
  - a face index out of range (Mesh.export's ValueError) and a writer error are raised by the next visualize() or
    flush(); that frame's file and the ones queued after it are not written;
  - the directory is made with os.makedirs instead of a shell running `mkdir -p`.
A DeviceMesh's file is byte for byte the one Mesh.export writes for the same vertices and faces."""
import atexit
import os
import queue
import weakref

import torch

from neuralbody_b200 import capi, mcubes
from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.evaluators.if_nerf import _colored
from neuralbody_b200.lib.visualizers.frame_writer import SLOTS, _flush_at_exit
from neuralbody_b200.png_writer import PngWriter


class MeshSlot:
    """The host side of one queued frame: `idx` (frame_index) int64, and either `out` (a DeviceMesh's packed buffer:
    status record, then the body of `nv` vertices and `nf` faces) or `mesh`, a host mesh."""

    def __init__(self, pin=True):
        self.pin = pin
        self.out = torch.empty(0, dtype=torch.uint8)
        self.idx = torch.empty(1, dtype=torch.int64, pin_memory=pin)
        self.nv = self.nf = 0
        self.mesh = None
        self.event = None

    def reserve(self, nbytes):
        """A pinned buffer of at least nbytes; replaced (with an eighth more room) only when the current one is smaller."""
        if self.out.numel() < nbytes:
            self.out = torch.empty(nbytes + nbytes // 8, dtype=torch.uint8, pin_memory=self.pin)
        return self.out[:nbytes]


class Visualizer:
    def __init__(self):
        cfg = get_active_cfg()
        print(_colored('the results are saved at {}'.format(os.path.join(cfg.result_dir, 'mesh')), 'yellow'))
        self._writer = PngWriter(depth=SLOTS, name="vis-mesh-writer")
        self._free = queue.Queue()
        pin = torch.cuda.is_available()
        for _ in range(SLOTS):
            self._free.put(MeshSlot(pin))
        # registered after torch's own exit handlers, so it runs before them: the last frames reach the disk
        atexit.register(_flush_at_exit, weakref.ref(self))

    def flush(self):
        """Wait until every queued frame's PLY file is written; raise the first error of any of them."""
        self._writer.join()

    def visualize(self, output, batch):
        cfg = get_active_cfg()
        self._writer.check()
        mesh = output['mesh']
        frame_index = batch['frame_index']
        result_dir = os.path.join(cfg.result_dir, 'mesh')
        slot = self._free.get()      # back-pressure: waits while every slot is queued
        try:
            stream = None
            if isinstance(mesh, mcubes.DeviceMesh):
                out = mesh.pack()
                slot.reserve(out.numel()).copy_(out, non_blocking=True)
                slot.nv, slot.nf = mesh.nv, mesh.nf
                stream = torch.cuda.current_stream(mesh.device)
            else:
                slot.mesh = mesh
            fi = torch.as_tensor(frame_index).reshape(-1)[:1]
            if fi.is_cuda:
                slot.idx.copy_(fi, non_blocking=True)
                stream = torch.cuda.current_stream(fi.device)
            else:
                slot.idx.copy_(fi)
            if stream is not None:
                if slot.event is None:
                    slot.event = torch.cuda.Event()
                slot.event.record(stream)
            event = slot.event if stream is not None else None
        except BaseException:
            slot.mesh = None
            self._free.put(slot)
            raise
        self._enqueue(slot, result_dir, event)

    def _enqueue(self, slot, result_dir, event):
        """Queue the writer's job for a filled slot, run after `event`; the slot is free again once the job is done or
        skipped."""
        free = self._free

        def write():
            if slot.mesh is None:
                mcubes.check_ply(slot.out.numpy())
            path = os.path.join(result_dir, '{:04d}.ply'.format(int(slot.idx[0])))
            os.makedirs(result_dir, exist_ok=True)
            if slot.mesh is not None:
                slot.mesh.export(path)
            else:
                body = slot.out.numpy()[capi.NB_MESH_PLY_BODY_OFFSET:capi.NB_MESH_PLY_BODY_OFFSET + 24 * slot.nv + 13 * slot.nf]
                with open(path, "wb") as f:
                    f.write(mcubes.ply_header(slot.nv, slot.nf))
                    f.write(body)

        def done():
            slot.mesh = None
            free.put(slot)

        self._writer.submit(write, event, done)
