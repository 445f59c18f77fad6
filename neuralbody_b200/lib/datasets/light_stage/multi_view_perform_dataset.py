"""Drop-in for the reference's novel-pose dataset lib/datasets/light_stage/multi_view_perform_dataset.py (selected through
`test_dataset_module / test_dataset_path` in `novel_pose_cfg`, for `run.py --type visualize` with `vis_novel_pose True`).

As multi_view_demo_dataset's drop-in: the item carries the render camera `cam_RT` = render_w2c[index % len(render_w2c)]
(4,4), `cam_K` (3,3) in upstream's dtype and the float32 `can_bounds` in place of upstream's host-built rays (:148-149),
and neuralbody_b200's renderers generate the rays on the GPU. `meta` holds the same three arrays: upstream's visualize
loop (run.py) moves every key but `meta` to the GPU, so the renderer reads the camera there with no copy back to the
host. Every other key is upstream's. The frame changes with every item here, so the masks (upstream's own get_mask and
resize) are built per item, as upstream builds them.  With `dataset_image_steps: 'device'` the item ships the decoded
`msks_u8` and the recipe under `meta` in place of `msks`, as multi_view_demo_dataset's drop-in does.

`make_dataset_class(base)` builds the subclass over any base with the reference's attributes (`K`, `Ks`, `RT`,
`render_w2c`, `prepare_input`, `get_mask`, and for the 'device' items `data_root`, `ims`, `Ds`); `Dataset` is the one
over the reference's own Dataset, resolved on first use.
The module name in `test_dataset_module` must be this module's
(`neuralbody_b200.lib.datasets.light_stage.multi_view_perform_dataset`), not upstream's, which it loads."""
import importlib

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import train_item
from neuralbody_b200.lib.datasets.light_stage.multi_view_demo_dataset import _cv2, _imread, decoded_masks, resized_masks

REFERENCE_MODULE = "lib.datasets.light_stage.multi_view_perform_dataset"


def make_dataset_class(base, cv2=None, imread=None):
    """-> a subclass of `base` whose __getitem__ returns the render camera in place of the rays (`cv2` and `imread` as in
    multi_view_demo_dataset.make_dataset_class)."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            # multi_view_perform_dataset.py:130-146
            frame_index = index + cfg.begin_ith_frame
            latent_index = index
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(frame_index)
            H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
            if train_item.image_steps(cfg) == 'device':
                msks, mask_meta = decoded_masks(self, index, H, W, imread if imread is not None else _imread)
            else:
                msks, mask_meta = {'msks': resized_masks(cv, self.get_mask(index), H, W)}, {}
            cam_ind = index % len(self.render_w2c)
            ret = {'coord': coord, 'out_sh': out_sh}
            # :161-174
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            latent_index = min(latent_index, cfg.num_train_frame - 1)
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index, 'frame_index': frame_index,
                        'view_index': cam_ind})
            ret.update(msks)
            ret.update({'Ks': self.Ks, 'RT': self.RT})
            # what image_rays (:148-149) reads
            ret.update({'cam_RT': self.render_w2c[cam_ind], 'cam_K': self.K, 'can_bounds': can_bounds})
            # a host copy for the renderer: upstream's visualize loop moves every key but 'meta' to the GPU
            ret['meta'] = {'cam_RT': ret['cam_RT'], 'cam_K': ret['cam_K'], 'can_bounds': can_bounds}
            ret['meta'].update(mask_meta)
            return ret

    return Dataset


_dataset = None


def __getattr__(name):
    """`Dataset`, over the reference's Dataset, built on first use."""
    global _dataset
    if name != "Dataset":
        raise AttributeError("module %r has no attribute %r" % (__name__, name))
    if _dataset is None:
        ref = importlib.import_module(REFERENCE_MODULE)
        if getattr(ref, "make_dataset_class", None) is make_dataset_class:
            raise ImportError("%s resolved to this drop-in: set test_dataset_module to "
                              "'neuralbody_b200.lib.datasets.light_stage.multi_view_perform_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
