"""Drop-in for the reference's People-Snapshot mesh dataset lib/datasets/light_stage/monocular_mesh_dataset.py (selected
through `test_dataset_module / test_dataset_path` in `mesh_cfg`, for `run.py --type visualize` with `vis_mesh True`).

Upstream's item carries the world grid `pts` (X,Y,Z,3) and its mask test `inside` (X,Y,Z), built on the host for every
frame (:78-90).  This item carries what that test reads instead, with a leading view dimension of 1: the frame's mask
`msks` (1,H,W) uint8 after upstream's own `cv2.undistort` and `INTER_NEAREST` resize by `cfg.ratio` (both stay on the
host), the intrinsics `Ks` (1,3,3) after upstream's `K[:2] * cfg.ratio`, and `RT = [R | T]` (1,3,4), the camera exactly as
prepare_inside_pts (:35-48) receives it -- float64 with upstream's `snapshot_data_utils.get_camera`, so the renderer
projects the grid in double (nb_mesh_inside_f64) as numpy does.  `wbounds` is upstream's float32 `can_bounds`.  The other
keys are upstream's: coord, out_sh, bounds, R, Th, latent_index (not clamped, as upstream), frame_index.
neuralbody_b200's if_mesh_renderer builds the grid axes and the test from them and returns the same cube and mesh.

The image is neither decoded nor resized: nothing downstream of the mesh item reads it.  The output size is therefore
taken from the mask, which has the image's size in People-Snapshot (upstream takes it from the image).

With `dataset_image_steps: 'device'` (default 'host') the item stops after decoding the mask: it ships `msks_u8`
(1,H0,W0) uint8 as read in place of `msks`, and the camera K, D and the recipe (no binarisation, no dilation, the
INTER_NEAREST resize by cfg.ratio) under `meta` (lib/datasets/mask_item.py); the mesh renderer builds the same `msks` on
the GPU (Renderer.mask_views, nb_mask_views).

`Dataset` subclasses the reference's own Dataset, resolved when it is first asked for (so this module imports without the
reference tree); `make_dataset_class(base)` builds the same subclass over any base with the reference's attributes
(`data_root`, `cam`, `begin_ith_frame`, `prepare_input`).  OpenCV and imageio are imported only when an item is built.
The module name in `test_dataset_module` must be this module's
(`neuralbody_b200.lib.datasets.light_stage.monocular_mesh_dataset`), not upstream's, which it loads."""
import importlib
import os

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import mask_item, train_item

REFERENCE_MODULE = "lib.datasets.light_stage.monocular_mesh_dataset"


def _cv2():
    import cv2
    return cv2


def _imread(path):
    import imageio
    return imageio.imread(path)


def make_dataset_class(base, cv2=None, imread=None):
    """-> a subclass of `base` whose __getitem__ returns the mask view in place of `pts` / `inside`.  `cv2`: the module
    providing undistort, resize, INTER_NEAREST and Rodrigues (OpenCV, imported on first use, when None); `imread`: the mask
    reader (imageio.imread, as upstream, when None)."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            read = imread if imread is not None else _imread
            # monocular_mesh_dataset.py:50-70
            latent_index = index
            index = index + self.begin_ith_frame
            frame_index = index
            msk = read(os.path.join(self.data_root, 'mask', '{}.png'.format(index)))
            K = self.cam['K']
            D = self.cam['D']
            device = train_item.image_steps(cfg) == 'device'
            if not device:
                msk = cv.undistort(msk, K, D)
            R = self.cam['R']
            T = self.cam['T'][:, None]
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(index)
            # :72-79, without the image
            H, W = int(msk.shape[0] * cfg.ratio), int(msk.shape[1] * cfg.ratio)
            if device:
                msk_keys, mask_meta = mask_item.mask_fields([msk], [K], [D], H, W, False, 0)
            else:
                msk = cv.resize(msk, (W, H), interpolation=cv.INTER_NEAREST)
                msk_keys, mask_meta = {'msks': np.asarray(msk, dtype=np.uint8)[None]}, None
            K = K.copy()
            K[:2] = K[:2] * cfg.ratio
            ret = {'coord': coord, 'out_sh': out_sh}
            # :95-104
            R_smpl = cv.Rodrigues(Rh)[0].astype(np.float32)
            ret.update({'wbounds': can_bounds, 'bounds': bounds, 'R': R_smpl, 'Th': Th, 'latent_index': latent_index,
                        'frame_index': frame_index})
            # what prepare_inside_pts (:35-48) reads: one view, the camera in its own dtype
            ret.update(msk_keys)
            ret['Ks'] = K[None]
            ret['RT'] = np.concatenate([R, T], axis=1)[None]
            if mask_meta is not None:
                ret['meta'] = mask_meta
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
                              "'neuralbody_b200.lib.datasets.light_stage.monocular_mesh_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
