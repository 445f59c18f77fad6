"""Drop-in for the reference's mesh renderer lib/networks/renderer/if_mesh_renderer.py (selected through
`renderer_module / renderer_path` for `run.py --type visualize` with `vis_mesh True`): density on the dataset's world
grid -> cube -> marching cubes at `cfg.mesh_th`, all on the GPU.

Same contract as upstream's `render(batch)` (:26-56): `batch['pts']` (1,X,Y,Z,3) world grid and `batch['inside']`
(1,X,Y,Z) uint8 from lib/datasets/light_stage/multi_view_mesh_dataset.py:121-160; the inside points' raw sigma (no relu)
is scattered into a zero cube, padded by 10 on every side, and returned as `'cube'` (host float64 numpy, upstream's
shape) with `'mesh'`, whose vertices are in padded index coordinates, as upstream leaves them.  B = 1, as upstream.

Differences to upstream: the inside points go through ONE density launch (nb_decode_density; upstream chunks by
2048 * 64 to bound PyTorch memory, which the kernel does not need), the cube stays on the device until the final copy,
and marching cubes is this package's kernel (neuralbody_b200/mcubes.py), not PyMCubes: the same edge crossings
interpolated the same way in double, but a watertight triangulation and grid-ordered output.  `'mesh'` is
`trimesh.Trimesh(vertices, triangles)` when trimesh is importable (upstream's call), else neuralbody_b200.mcubes.Mesh,
which has what lib/visualizers/if_nerf_mesh.py uses (`.vertices`, `.faces`, `.export(path)` as binary PLY)."""
import torch

from neuralbody_b200 import mcubes
from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.networks.renderer import if_nerf_renderer

PAD = 10   # np.pad(cube, 10) of if_mesh_renderer.py:47


class Renderer(if_nerf_renderer.Renderer):
    def __init__(self, net):
        super(Renderer, self).__init__(net)

    def density_cube(self, batch):
        """The padded density cube on the device (fp32: it holds the fp32 sigma and zeros, so it is exact as upstream's
        float64 cube), shape (X + 20, Y + 20, Z + 20)."""
        for k in ('pts', 'inside'):
            if k not in batch:
                raise KeyError("the mesh renderer needs batch['%s'] (lib/datasets/light_stage/multi_view_mesh_dataset.py:"
                               "150-169: the world grid 'pts' (1,X,Y,Z,3) and its mask-view test 'inside' (1,X,Y,Z))" % k)
        pts, inside = batch['pts'], batch['inside']
        if pts.device.type != "cuda" or inside.device.type != "cuda":
            raise RuntimeError("the mesh renderer needs CUDA tensors: there is no CPU implementation")
        if pts.dim() != 5 or pts.shape[0] != 1 or pts.shape[-1] != 3 or tuple(inside.shape) != tuple(pts.shape[:-1]):
            raise ValueError("batch['pts'] must be (1,X,Y,Z,3) and batch['inside'] (1,X,Y,Z) (B = 1, as upstream); got %s and %s"
                             % (tuple(pts.shape), tuple(inside.shape)))
        inside = inside[0].bool()
        wpts = pts[0][inside][None]
        sp_input = self.prepare_sp_input(batch)
        feature_volume = self.net.encode_sparse_voxels(sp_input)
        with torch.no_grad():
            alpha = self.net.calculate_density(wpts, feature_volume, sp_input)     # one nb_decode_density launch
            cube = torch.zeros(tuple(s + 2 * PAD for s in inside.shape), dtype=torch.float32, device=pts.device)
            cube[PAD:-PAD, PAD:-PAD, PAD:-PAD][inside] = alpha[0, :, 0]
        return cube

    def render(self, batch):
        cfg = get_active_cfg()
        cube = self.density_cube(batch)
        verts, tris = mcubes.marching_cubes(cube, float(cfg.mesh_th))
        mesh = mcubes.make_mesh(verts.cpu().numpy(), tris.cpu().numpy())
        return {'cube': cube.cpu().numpy().astype('float64'), 'mesh': mesh}
