"""Drop-in for the reference's rotate-SMPL dataset lib/datasets/light_stage/rotate_smpl_dataset.py (selected through
`test_dataset_module / test_dataset_path` in `rotate_smpl_cfg`, for `run.py --type visualize` with `vis_rotate_smpl True`).

As multi_view_demo_dataset's drop-in: upstream's item carries the view's rays, built on the host by render_utils.image_rays
for every one of its 144 views (:170-171); this item carries the render camera instead: `cam_RT` = render_w2c[0] (4,4)
and `cam_K` = the dataset's K (3,3), in the dtype upstream hands them to image_rays (float64 with ZJU-MoCap's
annotations), and `can_bounds` (2,3) float32, the rotated body's box.  neuralbody_b200's renderers generate the same rays,
near, far and mask_at_box from them on the GPU (Renderer.camera_rays).  `meta` holds the same three arrays: upstream's
visualize loop (run.py) moves every key but `meta` to the GPU, so the renderer reads the camera there with no copy back to
the host.  Every other key is upstream's, from upstream's own prepare_input(frame_index, view_index) on the host: coord,
out_sh, bounds, R, Th, latent_index, frame_index, view_index.

`make_dataset_class(base)` builds the subclass over any base with the reference's attributes (`K`, `render_w2c`,
`prepare_input`); `Dataset` is the one over the reference's own Dataset, resolved on first use.  The module name in
`test_dataset_module` must be this module's (`neuralbody_b200.lib.datasets.light_stage.rotate_smpl_dataset`), not
upstream's, which it loads."""
import importlib

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets.light_stage.multi_view_demo_dataset import _cv2

REFERENCE_MODULE = "lib.datasets.light_stage.rotate_smpl_dataset"


def make_dataset_class(base, cv2=None):
    """-> a subclass of `base` whose __getitem__ returns the render camera in place of the rays (`cv2` as in
    multi_view_demo_dataset.make_dataset_class)."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            # rotate_smpl_dataset.py:158-164
            i = cfg.ith_frame
            latent_index = i
            frame_index = i + cfg.begin_ith_frame
            view_index = index
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(frame_index, view_index)
            ret = {'coord': coord, 'out_sh': out_sh}
            # :183-193
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            latent_index = min(latent_index, cfg.num_train_frame - 1)
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index, 'frame_index': frame_index,
                        'view_index': view_index})
            # what image_rays (:170-171) reads
            ret.update({'cam_RT': self.render_w2c[0], 'cam_K': self.K, 'can_bounds': can_bounds})
            # a host copy for the renderer: upstream's visualize loop moves every key but 'meta' to the GPU
            ret['meta'] = {'cam_RT': ret['cam_RT'], 'cam_K': ret['cam_K'], 'can_bounds': can_bounds}
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
                              "'neuralbody_b200.lib.datasets.light_stage.rotate_smpl_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
