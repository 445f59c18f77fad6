"""Drop-in for the reference's People-Snapshot demo dataset lib/datasets/light_stage/monocular_demo_dataset.py (selected
through `test_dataset_module / test_dataset_path` in snapshot_f3c.yaml's novel-view / novel-pose settings).

Upstream's item carries the view's rays, built on the host by render_utils.image_rays (:113-114). This item carries the
camera that call reads instead: `cam_RT` = [R | T] (3,4) and `cam_K` (3,3), float32 as upstream casts them (:109-112),
and the float32 `can_bounds` (2,3) of the rotated body. neuralbody_b200's renderers generate the same rays, near, far
and mask_at_box from them on the GPU (nb_image_rays). `meta` holds the same three arrays: upstream's visualize loop
(run.py) moves every key but `meta` to the GPU, so the renderer reads the camera there with no copy back to the host.
Every other key is upstream's, including the mask `msk` (decoded, undistorted and resized on the host by upstream's own
calls) and `RT` / `K`, the same camera as the masked renderer reads it.  With `dataset_image_steps: 'device'` the item
stops after decoding the mask: it ships `msks_u8` (1,H0,W0) uint8 as read in place of `msk`, and the camera K, D and the
recipe (no binarisation, no dilation, the INTER_NEAREST resize by cfg.ratio) under `meta`; the `_msk` renderer builds
the same `msk` on the GPU (Renderer.mask_views, nb_mask_views).

`make_dataset_class(base)` builds the subclass over any base with the reference's attributes (`data_root`, `cam`,
`params`, `prepare_input`); `Dataset` is the one over the reference's own Dataset, resolved on first use.  OpenCV and
imageio are imported only when an item is built.  The module name in `test_dataset_module` must be this module's
(`neuralbody_b200.lib.datasets.light_stage.monocular_demo_dataset`), not upstream's, which it loads."""
import importlib
import os

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import mask_item, train_item

REFERENCE_MODULE = "lib.datasets.light_stage.monocular_demo_dataset"


def _cv2():
    import cv2
    return cv2


def _imread(path):
    import imageio
    return imageio.imread(path)


def make_dataset_class(base, cv2=None, imread=None):
    """-> a subclass of `base` whose __getitem__ returns the render camera in place of the rays.  `cv2`: the module
    providing undistort, resize, INTER_NEAREST and Rodrigues (OpenCV when None); `imread`: the mask reader (imageio.imread,
    as upstream, when None)."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            read = imread if imread is not None else _imread
            # monocular_demo_dataset.py:89-112
            K = self.cam['K']
            D = self.cam['D']
            R = self.cam['R']
            T = self.cam['T'][:, None]
            i = 0
            frame_index = i
            latent_index = i
            view_index = index
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(i, index)
            msk = read(os.path.join(self.data_root, 'mask', '{}.png'.format(i)))
            H, W = int(msk.shape[0] * cfg.ratio), int(msk.shape[1] * cfg.ratio)
            if train_item.image_steps(cfg) == 'device':
                msk_keys, mask_meta = mask_item.mask_fields([msk], [K], [D], H, W, False, 0)
            else:
                msk = cv.undistort(msk, K, D)
                msk = cv.resize(msk, (W, H), interpolation=cv.INTER_NEAREST)
                msk_keys, mask_meta = {'msk': msk}, {}
            K = K.copy().astype(np.float32)
            K[:2] = K[:2] * cfg.ratio
            RT = np.concatenate([R, T], axis=1).astype(np.float32)
            # :116-142 without the rays
            ret = {'coord': coord, 'out_sh': out_sh}
            ret.update(msk_keys)
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index, 'frame_index': frame_index,
                        'view_index': view_index})
            Rh0 = self.params['pose'][i][:3]
            R0 = cv.Rodrigues(Rh0)[0].astype(np.float32)
            Th0 = self.params['trans'][i].astype(np.float32)
            ret.update({'R0_snap': R0, 'Th0_snap': Th0, 'K': K, 'RT': RT})
            # what image_rays (:113-114) reads
            ret.update({'cam_RT': RT, 'cam_K': K, 'can_bounds': can_bounds})
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
                              "'neuralbody_b200.lib.datasets.light_stage.monocular_demo_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
