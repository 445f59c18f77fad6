"""Drop-in for the reference's single-view masked renderer lib/networks/renderer/if_clight_renderer_msk.py (selected by
configs/snapshot_exp/snapshot_f3c.yaml:88-89,105-106 for the People-Snapshot novel-view / novel-pose demos): a sample is
taken from the world to the SMPL frame with the rendered frame's (R, Th), from there into the world of the snapshot frame
with (`batch['R0_snap']`, `batch['Th0_snap']`), projected with that frame's camera (`batch['RT'] (1,3,4)`,
`batch['K'] (1,3,3)`) and kept only where `batch['msk'] (1,H,W)` is foreground; `raw` is 0 elsewhere (:12-49 and the
inherited if_clight_renderer_mmsk.py:47-94).

The predicate is one more test in the fused pipeline's sample classifier (nb_render_args.mask_R0 / mask_Th0): a
masked-out sample has sigma = 0, hence compositing weight exactly 0, and is skipped like an empty-space sample.
B = 1, as upstream."""
import torch

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.networks.renderer import if_nerf_renderer_mmsk


class Renderer(if_nerf_renderer_mmsk.Renderer):
    MASK_VIEWS_KEY = 'msk'

    def __init__(self, net):
        super(Renderer, self).__init__(net)

    def prepare_inside_pts(self, wpts, batch):
        """if_clight_renderer_msk.py:12-49 (host API parity; `render` evaluates the same predicate in-kernel)."""
        cfg = get_active_cfg()
        can_pts = torch.matmul(wpts - batch['Th'][:, None, None], batch['R'])
        sh = can_pts.shape
        can_pts = can_pts.view(sh[0], -1, sh[3])
        pts = torch.matmul(can_pts, batch['R0_snap'].transpose(2, 1)) + batch['Th0_snap'][:, None]
        pts = torch.matmul(pts, batch['RT'][..., :3].transpose(2, 1)) + batch['RT'][..., 3][:, None]
        pts = torch.matmul(pts, batch['K'].transpose(2, 1))
        pts2d = (pts[..., :2] / pts[..., 2:]).round().long()
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        pts2d[..., 0] = torch.clamp(pts2d[..., 0], 0, W - 1)
        pts2d[..., 1] = torch.clamp(pts2d[..., 1], 0, H - 1)
        pts2d = pts2d[0]
        return batch['msk'][0][pts2d[:, 1], pts2d[:, 0]][None].bool()

    def get_pixel_value(self, ray_o, ray_d, near, far, feature_volume, sp_input, batch):
        """if_clight_renderer_mmsk.py:63-94 with the single-view predicate above.  A batch of 'device' items carries the
        decoded view (`msks_u8`) in place of `msk`: mask_views builds it on the device first.  With `cfg.render_importance > 0`
        both passes of `render_rays_hierarchical` take the view, the snapshot transform included."""
        if 'msk' not in batch and 'msks_u8' in batch:
            self.mask_views(batch)
        for k in ('R0_snap', 'Th0_snap', 'RT', 'K', 'msk'):
            if k not in batch:
                raise KeyError("the single-view masked renderer needs batch['%s'] "
                               "(lib/datasets/light_stage/monocular_demo_dataset.py:138-141)" % k)
        cfg = get_active_cfg()
        H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
        if tuple(batch['msk'].shape[-2:]) != (H, W):
            raise ValueError("batch['msk'] is %s but cfg.H*ratio x cfg.W*ratio = %dx%d" % (tuple(batch['msk'].shape), H, W))
        masks = {"msks": batch['msk'][:, None], "RT": batch['RT'][:, None], "Ks": batch['K'][:, None],
                 "R0_snap": batch['R0_snap'], "Th0_snap": batch['Th0_snap']}
        if int(self._opt("render_importance", 0)) > 0:
            return self.render_rays_hierarchical(ray_o, ray_d, near, far, feature_volume, sp_input, masks=masks)
        return self.render_rays(ray_o, ray_d, near, far, feature_volume, sp_input, masks=masks)
