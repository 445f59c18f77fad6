"""Drop-in for the reference's lib/train/trainers/if_nerf_clight.py, selected from the yaml alone: upstream's
make_trainer._wrapper_factory loads `NetworkWrapper` from `cfg.trainer_path` (module name `cfg.trainer_module`), so

    trainer_module: 'lib.train.trainers.if_nerf_clight'
    trainer_path: '<this package>/lib/train/trainers/if_nerf_clight.py'

trains through upstream's train_net.py unchanged.  Same class, constructor, attributes (`net`, `renderer`) and
`forward(batch) -> (ret, loss, scalar_stats, image_stats)` with the same keys (`img_loss`, `img_loss0` when the render
returns `rgb0`, `loss`).  Two differences, neither visible in the results:
  - the renderer is this package's if_nerf_renderer.Renderer (upstream hard-imports if_clight_renderer);
  - the two image losses run on the device (neuralbody_b200.image_loss, nb_image_loss_fwd / _bwd) instead of
    torch.mean((rgb_map[mask] - rgb[mask]) ** 2), whose boolean index is a nonzero: the host would wait there for the
    whole forward pass before queuing the backward.  The loss is the float64 sum rounded once; its gradient is autograd's
    for upstream's expression, bit for bit.
It takes upstream's training items and this package's (`img` / `train_cam`, `dataset_image_steps: 'device'`): the renderer
writes `rgb` and `mask_at_box` into a batch that ships the image, before the loss reads them.  Under torch.no_grad()
(Trainer.val) the same forward returns upstream's stats.  A mask whose shape differs from the rays' raises IndexError, as
upstream's index does (a test-split view whose rays do not fill the image)."""
import torch
import torch.nn as nn

from neuralbody_b200.image_loss import image_mse
from neuralbody_b200.lib.networks.renderer import if_nerf_renderer


class NetworkWrapper(nn.Module):
    def __init__(self, net):
        super(NetworkWrapper, self).__init__()

        self.net = net
        self.renderer = if_nerf_renderer.Renderer(self.net)

        self.img2mse = image_mse
        self.acc_crit = torch.nn.functional.smooth_l1_loss

    def forward(self, batch):
        ret = self.renderer.render(batch)

        scalar_stats = {}
        loss = 0

        mask = batch['mask_at_box']
        img_loss = self.img2mse(ret['rgb_map'], batch['rgb'], mask)
        scalar_stats.update({'img_loss': img_loss})
        loss += img_loss

        if 'rgb0' in ret:
            img_loss0 = self.img2mse(ret['rgb0'], batch['rgb'])
            scalar_stats.update({'img_loss0': img_loss0})
            loss += img_loss0

        scalar_stats.update({'loss': loss})
        image_stats = {}

        return ret, loss, scalar_stats, image_stats
