"""Drop-in for the reference's masked renderer lib/networks/renderer/if_clight_renderer_mmsk.py (the renderer
behind `vis_novel_view` / `vis_novel_pose`, lib/config/config.py:157-167): every sample is projected into the
`nv` training-view masks (`batch['RT'] (1,nv,3,4)`, `batch['Ks'] (1,nv,3,3)`, `batch['msks'] (1,nv,H,W)`); the
decoder runs only where all masks are foreground and `raw` is 0 elsewhere (:47-61).

Here the predicate is evaluated inside the fused kernel's sample classifier: a masked-out sample has sigma = 0,
hence compositing weight exactly 0, so it is skipped exactly like an empty-space sample.  B = 1, as upstream."""
import torch

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.networks.renderer import if_nerf_renderer


class Renderer(if_nerf_renderer.Renderer):
    def __init__(self, net):
        super(Renderer, self).__init__(net)

    def prepare_inside_pts(self, pts, batch):
        """if_clight_renderer_mmsk.py:12-45 (host API parity; `render` evaluates the same predicate in-kernel)."""
        cfg = get_active_cfg()
        sh = pts.shape
        pts = pts.view(sh[0], -1, sh[3])
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        inside = None
        for nv in range(batch['Ks'].size(1)):
            R = batch['RT'][:, nv, :3, :3]
            T = batch['RT'][:, nv, :3, 3]
            pts_ = torch.matmul(pts, R.transpose(2, 1)) + T[:, None]
            pts_ = torch.matmul(pts_, batch['Ks'][:, nv].transpose(2, 1))
            pts2d = (pts_[..., :2] / pts_[..., 2:]).round().long()
            pts2d[..., 0] = torch.clamp(pts2d[..., 0], 0, W - 1)
            pts2d[..., 1] = torch.clamp(pts2d[..., 1], 0, H - 1)
            pts2d = pts2d[0]
            ins = batch['msks'][0, nv][pts2d[:, 1], pts2d[:, 0]][None].bool()
            inside = ins if inside is None else inside * ins
        return inside

    def get_pixel_value(self, ray_o, ray_d, near, far, feature_volume, sp_input, batch):
        """if_clight_renderer_mmsk.py:63-94.  A batch of 'device' items carries the decoded views (`msks_u8`) in place of
        `msks`: mask_views builds them on the device first.  With `cfg.render_importance > 0` the view gets the coarse + fine
        passes of `render_rays_hierarchical`, both masked, and the dict also carries rgb0 / disp0 / acc0 / z_std."""
        if 'msks' not in batch and 'msks_u8' in batch:
            self.mask_views(batch)
        if 'Ks' not in batch or 'RT' not in batch or 'msks' not in batch:
            raise KeyError("the masked renderer needs batch['RT'], batch['Ks'] and batch['msks'] "
                           "(lib/datasets/light_stage/multi_view_demo_dataset.py:107-129)")
        cfg = get_active_cfg()
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        if tuple(batch['msks'].shape[-2:]) != (H, W):
            raise ValueError("batch['msks'] is %s but cfg.H*ratio x cfg.W*ratio = %dx%d" % (tuple(batch['msks'].shape), H, W))
        if int(self._opt("render_importance", 0)) > 0:
            return self.render_rays_hierarchical(ray_o, ray_d, near, far, feature_volume, sp_input, masks=batch)
        return self.render_rays(ray_o, ray_d, near, far, feature_volume, sp_input, masks=batch)
