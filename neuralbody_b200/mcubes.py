"""Marching cubes on the GPU (nb_mcubes_count / nb_mcubes_emit) and a minimal triangle mesh with a binary PLY writer.

`marching_cubes(volume, isovalue)` mirrors `mcubes.marching_cubes` (PyMCubes), the call of the reference's mesh renderer
(lib/networks/renderer/if_mesh_renderer.py:48): vertices (V,3) float64 in index coordinates, triangles (F,3) int64.  It
takes and returns CUDA tensors; there is no CPU implementation.  The mesh is the same set of edge crossings,
interpolated the same way in double, but the triangulation is this package's own table (csrc/nb_mc_table.h): it
separates the inside corners of every ambiguous face, so the mesh is closed, and its vertex / triangle order is the
grid order, not PyMCubes'.

`Mesh` writes a mesh's binary PLY on the host; `DeviceMesh` keeps it on the device and packs the same PLY body there
(nb_mesh_ply), so the file takes one copy back; `ply_header` is the header both write."""
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


FACE_RANGE_ERROR = "face indices out of range for a PLY int32 list"


def ply_header(nv, nf):
    """The header of the binary little-endian PLY that Mesh.export and DeviceMesh.export write: nv double x y z vertices,
    nf faces as uchar-counted int32 index lists."""
    return ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty double x\nproperty double y\n"
            "property double z\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
            % (nv, nf)).encode("ascii")


def _write(file_obj, data):
    if hasattr(file_obj, "write"):
        file_obj.write(data)
    else:
        with open(file_obj, "wb") as f:
            f.write(data)


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
            raise ValueError(FACE_RANGE_ERROR)
        head = ply_header(len(self.vertices), len(self.faces))
        face_rec = np.empty(len(self.faces), dtype=np.dtype([("n", "u1"), ("idx", "<i4", (3,))]))
        face_rec["n"] = 3
        face_rec["idx"] = self.faces
        data = head + self.vertices.astype("<f8").tobytes() + face_rec.tobytes()
        _write(file_obj, data)
        return data


class DeviceMesh:
    """A marching-cubes mesh that stays on the device: `.vertices` (V,3) float64 and `.faces` (F,3) int64 CUDA tensors, and
    the host counts `nv` / `nf` (their shapes, known since marching cubes' count read).  `export(path_or_file)` writes the
    bytes `Mesh(vertices.cpu(), faces.cpu()).export` writes and raises its ValueError for a face index out of range, so the
    reference's mesh visualizer works with it unchanged; the body is packed on the device (nb_mesh_ply) and comes back in
    one copy.  `pack()` only enqueues, for callers that copy and write off the render loop
    (lib/visualizers/if_nerf_mesh.py)."""

    def __init__(self, vertices, faces):
        if not (torch.is_tensor(vertices) and torch.is_tensor(faces) and vertices.is_cuda and faces.device == vertices.device):
            raise ValueError("DeviceMesh needs vertices and faces as CUDA tensors on one device")
        if vertices.dtype != torch.float64 or faces.dtype != torch.int64 or vertices.dim() != 2 or faces.dim() != 2 or \
                vertices.shape[1] != 3 or faces.shape[1] != 3:
            raise ValueError("DeviceMesh needs vertices (V,3) float64 and faces (F,3) int64 (got %s %s and %s %s)"
                             % (tuple(vertices.shape), vertices.dtype, tuple(faces.shape), faces.dtype))
        self.vertices, self.faces = vertices.contiguous(), faces.contiguous()
        self.nv, self.nf = int(vertices.shape[0]), int(faces.shape[0])

    @property
    def device(self):
        return self.vertices.device

    def body_bytes(self):
        return 24 * self.nv + 13 * self.nf

    def pack(self):
        """Enqueue nb_mesh_ply on the current stream -> a device uint8 tensor: the nb_mesh_ply_result record, then from
        capi.NB_MESH_PLY_BODY_OFFSET the PLY body.  A mesh whose vertices Mesh.export refuses (V >= 2^31) with faces is its
        ValueError here; nothing synchronises with the host."""
        if self.nf and self.nv >= 2 ** 31:
            raise ValueError(FACE_RANGE_ERROR)
        lib = capi.load()
        dev = self.device
        with torch.cuda.device(dev):
            out = torch.empty(capi.NB_MESH_PLY_BODY_OFFSET + self.body_bytes(), dtype=torch.uint8, device=dev)
            a = capi.nb_mesh_ply_args()
            a.nv, a.nf = self.nv, self.nf
            a.vertices, a.faces = self.vertices.data_ptr() or None, self.faces.data_ptr() or None
            a.out, a.out_bytes = out.data_ptr(), out.numel()
            capi.check(lib.nb_mesh_ply(C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "nb_mesh_ply")
        return out

    def export(self, file_obj):
        """Write binary PLY to a path or a binary file object, byte for byte what Mesh.export writes for the host copy of
        this mesh; returns the bytes written.  Synchronises with the host (the body's copy)."""
        out = self.pack().cpu().numpy()
        check_ply(out)
        data = ply_header(self.nv, self.nf) + out[capi.NB_MESH_PLY_BODY_OFFSET:].tobytes()
        _write(file_obj, data)
        return data

    def cpu(self):
        """The host Mesh of the same vertices and faces."""
        return Mesh(self.vertices.cpu().numpy(), self.faces.cpu().numpy())


def check_ply(out_host):
    """The host copy of DeviceMesh.pack's buffer (uint8 numpy array): Mesh.export's ValueError when a face index is out of
    range."""
    r = capi.nb_mesh_ply_result.from_buffer_copy(np.asarray(out_host)[:C.sizeof(capi.nb_mesh_ply_result)].tobytes())
    if r.status != capi.NB_MESH_PLY_OK:
        raise ValueError(FACE_RANGE_ERROR)


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

