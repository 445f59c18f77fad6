"""Drop-in for the reference's mesh renderer lib/networks/renderer/if_mesh_renderer.py (selected through
`renderer_module / renderer_path` for `run.py --type visualize` with `vis_mesh True`): density on the dataset's world
grid -> cube -> marching cubes at `cfg.mesh_th`, all on the GPU.

Same contract as upstream's `render(batch)` (:26-56): `batch['pts']` (1,X,Y,Z,3) world grid and `batch['inside']`
(1,X,Y,Z) uint8 from lib/datasets/light_stage/multi_view_mesh_dataset.py:121-160.  A batch without them may carry the
frame's mask views instead (`wbounds` (1,2,3), `RT` (1,nv,3,4), `Ks` (1,nv,3,3), `msks` (1,nv,H,W), as this package's
drop-ins lib/datasets/light_stage/multi_view_mesh_dataset.py (float32 camera) and monocular_mesh_dataset.py (nv = 1,
float64 camera) return them): the grid's axes and its mask-view test are then built here, the test on the device in the
camera's precision, with the same result.  The inside points' raw sigma (no relu)
is scattered into a zero cube, padded by 10 on every side, and returned as `'cube'` (host float64 numpy, upstream's
shape) with `'mesh'`, whose vertices are in padded index coordinates, as upstream leaves them.  B = 1, as upstream.

Differences to upstream: the inside points go through ONE density launch (nb_decode_density; upstream chunks by
2048 * 64 to bound PyTorch memory, which the kernel does not need), the cube stays on the device until the final copy,
and marching cubes is this package's kernel (neuralbody_b200/mcubes.py), not PyMCubes: the same edge crossings
interpolated the same way in double, but a watertight triangulation and grid-ordered output.  `'mesh'` is
`trimesh.Trimesh(vertices, triangles)` when trimesh is importable (upstream's call), else neuralbody_b200.mcubes.Mesh,
which has what lib/visualizers/if_nerf_mesh.py uses (`.vertices`, `.faces`, `.export(path)` as binary PLY).

`cfg.mesh_output` (default 'host') picks where the outputs live.  'host' is upstream's contract above.  'device' leaves
both on the GPU, so render() copies neither back: `'cube'` is the padded fp32 CUDA tensor (its values are the host cube's
float64 values) and `'mesh'` a neuralbody_b200.mcubes.DeviceMesh, whose `.export(path)` writes the same PLY bytes and which
this package's lib/visualizers/if_nerf_mesh.py writes off the visualize loop.  What still waits on the device is the
inside points' selection (boolean indexing sizes its result; a mask-view batch also reads its world box) and marching
cubes' count read."""
import ctypes as C

import numpy as np
import torch

from neuralbody_b200 import capi, mcubes
from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.networks.renderer import if_nerf_renderer

PAD = 10   # np.pad(cube, 10) of if_mesh_renderer.py:47
MASK_KEYS = ('wbounds', 'RT', 'Ks', 'msks')
MESH_OUTPUTS = ('host', 'device')


def world_axes(wbounds, voxel_size):
    """multi_view_mesh_dataset.py:150-156: the x, y and z planes of the world grid (float32, as the grid's `pts`) over the
    float32 world box wbounds (2,3), spaced cfg.voxel_size.  This is numpy's own arange on the dataset's operands (a
    float32 bound, python floats), because its values follow numpy's scalar promotion: under NumPy 2 the second element
    start + step is a float32 sum and the fill step is its float64 difference from start, so a restated formula would
    not reproduce the dataset's grid."""
    wb = np.asarray(wbounds, dtype=np.float32)
    vs = [float(v) for v in voxel_size]
    return [np.arange(wb[0, a], wb[1, a] + vs[a], vs[a]).astype(np.float32) for a in range(3)]


def camera_is_f64(RT, Ks):
    """True for a float64 camera (both RT and Ks float64: the monocular mesh dataset's, projected in double by
    nb_mesh_inside_f64), False otherwise (projected in fp32 by nb_mesh_inside, the multi-view dataset's float32 camera).
    A camera with only one of the two in float64 is a ValueError: numpy would project it with a chain neither kernel
    reproduces."""
    f64 = (RT.dtype == torch.float64, Ks.dtype == torch.float64)
    if f64[0] != f64[1]:
        raise ValueError("the mask views' RT and Ks must both be float64 (projected in double) or neither; got %s and %s"
                         % (RT.dtype, Ks.dtype))
    return f64[0]


def grid_inside(axes, RT, Ks, msks):
    """prepare_inside_pts (multi_view_mesh_dataset.py:117-140, monocular_mesh_dataset.py:35-48) on the device, one launch:
    axes = the grid's x, y and z planes (CUDA fp32 vectors), RT (nv,3,4), Ks (nv,3,3), msks (nv,H,W) CUDA tensors on the
    same device.  A float64 camera is projected in double (nb_mesh_inside_f64), any other in fp32 (nb_mesh_inside); see
    `camera_is_f64`.  -> inside (X,Y,Z) uint8, the last mask value each point read (views in order, on while it reads
    exactly 1)."""
    if any(t.device.type != "cuda" for t in (RT, Ks, msks, *axes)):
        raise RuntimeError("grid_inside needs CUDA tensors: there is no CPU implementation")
    nv = int(msks.shape[0]) if msks.dim() == 3 else -1
    if nv < 1 or tuple(RT.shape) != (nv, 3, 4) or tuple(Ks.shape) != (nv, 3, 3) or any(a.dim() != 1 for a in axes):
        raise ValueError("grid_inside: msks must be (nv,H,W) with nv >= 1, RT (nv,3,4), Ks (nv,3,3) and the axes vectors; got "
                         "%s, %s, %s" % (tuple(msks.shape), tuple(RT.shape), tuple(Ks.shape)))
    f64 = camera_is_f64(RT, Ks)
    cam_dtype = torch.float64 if f64 else torch.float32
    dev = msks.device
    with torch.cuda.device(dev):
        x, y, z = (a.to(device=dev, dtype=torch.float32).contiguous() for a in axes)
        m = msks.to(torch.uint8).contiguous()
        rt = RT.to(cam_dtype).contiguous()
        ks = Ks.to(cam_dtype).contiguous()
        inside = torch.empty((len(x), len(y), len(z)), dtype=torch.uint8, device=dev)
        a = capi.nb_mesh_inside_args()
        a.x, a.y, a.z = x.data_ptr(), y.data_ptr(), z.data_ptr()
        a.nx, a.ny, a.nz = inside.shape
        a.msks, a.inside = m.data_ptr(), inside.data_ptr()
        a.nv, a.H, a.W = (int(s) for s in m.shape)
        lib = capi.load()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        if f64:
            capi.check(lib.nb_mesh_inside_f64(C.byref(a), rt.data_ptr(), ks.data_ptr(), stream), "nb_mesh_inside_f64")
        else:
            a.RT, a.Ks = rt.data_ptr(), ks.data_ptr()
            capi.check(lib.nb_mesh_inside(C.byref(a), stream), "nb_mesh_inside")
    return inside


def mesh_output(cfg):
    """cfg.mesh_output, read with its default 'host' (upstream's cfg has no such key); any value but MESH_OUTPUTS is a
    ValueError."""
    mode = cfg.get('mesh_output', 'host')
    if mode not in MESH_OUTPUTS:
        raise ValueError("cfg.mesh_output must be one of %s (got %r)" % (", ".join(repr(m) for m in MESH_OUTPUTS), mode))
    return mode


class Renderer(if_nerf_renderer.Renderer):
    def __init__(self, net):
        super(Renderer, self).__init__(net)

    def density_cube(self, batch):
        """The padded density cube on the device (fp32: it holds the fp32 sigma and zeros, so it is exact as upstream's
        float64 cube), shape (X + 20, Y + 20, Z + 20).  The grid comes from the batch's `pts` / `inside` when both are
        there, else from its mask views (`wbounds`, `RT`, `Ks`, `msks`; see `grid_from_masks`).  A batch of 'device' items
        carries the decoded views (`msks_u8`) in place of `msks`: mask_views builds them on the device first."""
        if 'pts' not in batch and 'msks' not in batch and 'msks_u8' in batch:
            self.mask_views(batch)
        if 'pts' in batch and 'inside' in batch:
            wpts, inside = self.grid_from_points(batch)
        elif all(k in batch for k in MASK_KEYS):
            wpts, inside = self.grid_from_masks(batch)
        else:
            raise KeyError("the mesh renderer needs either batch['pts'] (1,X,Y,Z,3) and batch['inside'] (1,X,Y,Z) (the world "
                           "grid and its mask-view test, lib/datasets/light_stage/multi_view_mesh_dataset.py:150-169) or "
                           "batch['wbounds'] (1,2,3), batch['RT'] (1,nv,3,4), batch['Ks'] (1,nv,3,3) and batch['msks'] "
                           "(1,nv,H,W) (the frame's mask views, neuralbody_b200/lib/datasets/light_stage/"
                           "multi_view_mesh_dataset.py); got keys %s" % sorted(batch))
        sp_input = self.prepare_sp_input(batch)
        feature_volume = self.net.encode_sparse_voxels(sp_input)
        with torch.no_grad():
            alpha = self.net.calculate_density(wpts, feature_volume, sp_input)     # one nb_decode_density launch
            cube = torch.zeros(tuple(s + 2 * PAD for s in inside.shape), dtype=torch.float32, device=wpts.device)
            cube[PAD:-PAD, PAD:-PAD, PAD:-PAD][inside] = alpha[0, :, 0]
        return cube

    def grid_from_points(self, batch):
        """Upstream's contract: -> (the inside points (1,n,3), inside (X,Y,Z) bool) from batch['pts'] / batch['inside']."""
        pts, inside = batch['pts'], batch['inside']
        if pts.device.type != "cuda" or inside.device.type != "cuda":
            raise RuntimeError("the mesh renderer needs CUDA tensors: there is no CPU implementation")
        if pts.dim() != 5 or pts.shape[0] != 1 or pts.shape[-1] != 3 or tuple(inside.shape) != tuple(pts.shape[:-1]):
            raise ValueError("batch['pts'] must be (1,X,Y,Z,3) and batch['inside'] (1,X,Y,Z) (B = 1, as upstream); got %s and %s"
                             % (tuple(pts.shape), tuple(inside.shape)))
        inside = inside[0].bool()
        return pts[0][inside][None], inside

    def grid_from_masks(self, batch):
        """The same (inside points, inside) from the frame's mask views, without the (X,Y,Z,3) grid: the axes on the host
        (`world_axes`), the mask-view test of prepare_inside_pts on the device (nb_mesh_inside, one launch), and the inside
        points gathered from the axes at inside.nonzero() -- the values and the order of pts[0][inside].  The camera's dtype
        picks the projection: float64 RT / Ks (the monocular dataset's) are projected in double, float32 ones in fp32."""
        wb, RT, Ks, msks = (batch[k] for k in MASK_KEYS)
        camera_is_f64(RT, Ks)
        if RT.device.type != "cuda" or Ks.device.type != "cuda" or msks.device.type != "cuda":
            raise RuntimeError("the mesh renderer needs CUDA tensors: there is no CPU implementation")
        nv = int(msks.shape[1]) if msks.dim() == 4 else -1
        if (msks.dim() != 4 or msks.shape[0] != 1 or nv < 1 or tuple(RT.shape) != (1, nv, 3, 4)
                or tuple(Ks.shape) != (1, nv, 3, 3) or tuple(wb.shape) != (1, 2, 3)):
            raise ValueError("batch['msks'] must be (1,nv,H,W) with nv >= 1, batch['RT'] (1,nv,3,4), batch['Ks'] (1,nv,3,3) and "
                             "batch['wbounds'] (1,2,3) (B = 1, as upstream); got %s, %s, %s and %s"
                             % (tuple(msks.shape), tuple(RT.shape), tuple(Ks.shape), tuple(wb.shape)))
        axes = [torch.from_numpy(a).to(msks.device) for a in world_axes(wb[0].detach().cpu().numpy(),
                                                                         get_active_cfg().voxel_size)]
        inside = grid_inside(axes, RT[0], Ks[0], msks[0]).bool()
        ijk = inside.nonzero()
        wpts = torch.stack([axes[0][ijk[:, 0]], axes[1][ijk[:, 1]], axes[2][ijk[:, 2]]], dim=1)
        return wpts[None], inside

    def render(self, batch):
        cfg = get_active_cfg()
        mode = mesh_output(cfg)
        cube = self.density_cube(batch)
        verts, tris = mcubes.marching_cubes(cube, float(cfg.mesh_th))
        if mode == 'device':
            return {'cube': cube, 'mesh': mcubes.DeviceMesh(verts, tris)}
        mesh = mcubes.make_mesh(verts.cpu().numpy(), tris.cpu().numpy())
        return {'cube': cube.cpu().numpy().astype('float64'), 'mesh': mesh}
