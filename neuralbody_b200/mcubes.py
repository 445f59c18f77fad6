"""Marching cubes on the GPU (nb_mcubes_count / nb_mcubes_emit) and a minimal triangle mesh with a binary PLY writer.

`marching_cubes(volume, isovalue)` mirrors `mcubes.marching_cubes` (PyMCubes), the call of the reference's mesh renderer
(lib/networks/renderer/if_mesh_renderer.py:48): vertices (V,3) float64 in index coordinates, triangles (F,3) int64.  It
takes and returns CUDA tensors; there is no CPU implementation.  The mesh is the same set of edge crossings,
interpolated the same way in double, but the triangulation is this package's own table (csrc/nb_mc_table.h): it
separates the inside corners of every ambiguous face, so the mesh is closed, and its vertex / triangle order is the
grid order, not PyMCubes'."""
import ctypes as C

import numpy as np
import torch

from . import capi


def marching_cubes(volume, isovalue):
    """volume: CUDA tensor (nx, ny, nz) (converted to contiguous fp32); isovalue: float; a value > isovalue is inside.
    Returns (vertices (V,3) float64, triangles (F,3) int64) on the volume's device.  One host sync (to size the outputs)."""
    if not isinstance(volume, torch.Tensor) or volume.dim() != 3:
        raise ValueError("marching_cubes expects a 3-d tensor (nx, ny, nz)")
    dev = volume.device
    if dev.type != "cuda":
        raise RuntimeError("marching_cubes needs a CUDA tensor: there is no CPU implementation")
    lib = capi.load()
    nx, ny, nz = (int(s) for s in volume.shape)
    with torch.cuda.device(dev):
        grid = volume.detach().to(torch.float32).contiguous()
        a = capi.nb_mcubes_args()
        a.grid, a.nx, a.ny, a.nz, a.isovalue = grid.data_ptr(), nx, ny, nz, float(isovalue)
        nbytes = int(lib.nb_mcubes_workspace_bytes(nx, ny, nz)) if min(nx, ny, nz) >= 1 else 0
        if nbytes == 0:
            # invalid dims or a grid beyond the 32-bit offsets: nb_mcubes_count reports which
            nbytes = 256
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        a.workspace, a.workspace_bytes, a.counts = ws.data_ptr(), nbytes, counts.data_ptr()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        capi.check(lib.nb_mcubes_count(C.byref(a), stream), "nb_mcubes_count")
        nv, nt = (int(x) for x in counts.tolist())
        verts = torch.empty((nv, 3), dtype=torch.float64, device=dev)
        tris = torch.empty((nt, 3), dtype=torch.int64, device=dev)
        if nv > 0 or nt > 0:
            a.vertices, a.triangles = verts.data_ptr(), tris.data_ptr()
            capi.check(lib.nb_mcubes_emit(C.byref(a), stream), "nb_mcubes_emit")
    return verts, tris


class Mesh:
    """The part of trimesh.Trimesh the reference's mesh visualizer uses (lib/visualizers/if_nerf_mesh.py:28-36):
    `.vertices`, `.faces` and `.export(path)`, which writes binary little-endian PLY (double x y z, int32 index lists).
    No processing: vertices and faces are kept as given."""

    def __init__(self, vertices, faces):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)

    def export(self, file_obj):
        """Write binary PLY to a path or a binary file object; returns the bytes written."""
        if len(self.faces) and (self.faces.min() < 0 or self.faces.max() >= max(len(self.vertices), 1) or
                                len(self.vertices) >= 2 ** 31):
            raise ValueError("face indices out of range for a PLY int32 list")
        head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty double x\nproperty double y\n"
                "property double z\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                % (len(self.vertices), len(self.faces))).encode("ascii")
        face_rec = np.empty(len(self.faces), dtype=np.dtype([("n", "u1"), ("idx", "<i4", (3,))]))
        face_rec["n"] = 3
        face_rec["idx"] = self.faces
        data = head + self.vertices.astype("<f8").tobytes() + face_rec.tobytes()
        if hasattr(file_obj, "write"):
            file_obj.write(data)
        else:
            with open(file_obj, "wb") as f:
                f.write(data)
        return data


def read_ply(path):
    """Read back a triangle mesh written by Mesh.export -> (vertices (V,3) float64, faces (F,3) int64)."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").split("\n")
    if header[1] != "format binary_little_endian 1.0":
        raise ValueError("not a binary little-endian PLY")
    nv = nf = None
    for line in header:
        if line.startswith("element vertex "):
            nv = int(line.split()[-1])
        elif line.startswith("element face "):
            nf = int(line.split()[-1])
    verts = np.frombuffer(data, dtype="<f8", count=3 * nv, offset=end).reshape(nv, 3).astype(np.float64)
    off = end + 24 * nv
    rec = np.frombuffer(data, dtype=np.dtype([("n", "u1"), ("idx", "<i4", (3,))]), count=nf, offset=off)
    if nf and (rec["n"] != 3).any():
        raise ValueError("only triangle faces are supported")
    if off + rec.nbytes != len(data):
        raise ValueError("trailing bytes after the face list: %d" % (len(data) - off - rec.nbytes))
    return verts, rec["idx"].astype(np.int64).reshape(nf, 3)


def make_mesh(vertices, faces):
    """trimesh.Trimesh(vertices, faces) when trimesh is importable -- the reference's own call -- else a `Mesh`."""
    try:
        import trimesh
    except ImportError:
        return Mesh(vertices, faces)
    return trimesh.Trimesh(vertices, faces)

