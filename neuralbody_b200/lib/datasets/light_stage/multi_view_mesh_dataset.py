"""Drop-in for the reference's mesh dataset lib/datasets/light_stage/multi_view_mesh_dataset.py (selected through
`test_dataset_module / test_dataset_path` in `mesh_cfg`, for `run.py --type visualize` with `vis_mesh True`).

Upstream's item carries the world grid `pts` (X,Y,Z,3) and its mask-view test `inside` (X,Y,Z), built on the host for
every frame (:142-181; 8.07 M points for the full-size ZJU-MoCap 313 body).  This item carries what that test reads
instead: the frame's training-view masks `msks` (nv,H,W) uint8 from upstream's own `get_mask` (undistorted and dilated on
the host, as before), the intrinsics `Ks` (nv,3,3) and the world->camera `RT = [R | T]` (nv,3,4) float32, T in metres,
as prepare_inside_pts builds it (:126).  The other keys are upstream's: coord, out_sh, wbounds, bounds, R, Th,
latent_index, frame_index.  neuralbody_b200's if_mesh_renderer builds the grid axes and the test from them, the test on
the GPU (nb_mesh_inside), and returns the same cube and mesh.

With `dataset_image_steps: 'device'` (default 'host') the item stops after decoding the masks: it ships `msks_u8`
(nv,H0,W0) uint8 as read, before upstream's binarisation, in place of `msks`, and each view's camera (`Ks[nv]` as stored,
`Ds[nv]`) and the recipe (binarise, 5 x 5 dilation, no resize) under `meta` (lib/datasets/mask_item.py); the mesh
renderer builds the same `msks` on the GPU (Renderer.mask_views, nb_mask_views).

`Dataset` subclasses the reference's own Dataset, resolved when it is first asked for (so this module imports without the
reference tree); `make_dataset_class(base)` builds the same subclass over any base with the reference's attributes
(`ims`, `Ks`, `Rs`, `Ts`, `prepare_input`, `get_mask`, and for the 'device' items `data_root`, `Ds`), and OpenCV is imported only when an item is built.  The module name in `test_dataset_module` must be this module's
(`neuralbody_b200.lib.datasets.light_stage.multi_view_mesh_dataset`), not upstream's, which it loads."""
import importlib

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import mask_item, train_item

REFERENCE_MODULE = "lib.datasets.light_stage.multi_view_mesh_dataset"


def _cv2_rodrigues(rvec):
    import cv2
    return cv2.Rodrigues(rvec)


def _imread(path):
    import imageio
    return imageio.imread(path)


def make_dataset_class(base, rodrigues=_cv2_rodrigues, imread=None):
    """-> a subclass of `base` whose __getitem__ returns the mask views in place of `pts` / `inside`.  `rodrigues`: the
    axis-angle -> (rotation matrix, jacobian) conversion of the item's R, cv2.Rodrigues as upstream calls it; `imread`: the
    mask reader of the 'device' items (imageio.imread, as upstream, when None)."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            # multi_view_mesh_dataset.py:143-148
            i = index
            latent_index = index
            frame_index = index + cfg.begin_ith_frame
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(frame_index)
            ret = {'coord': coord, 'out_sh': out_sh}
            # :169-181
            R = rodrigues(Rh)[0].astype(np.float32)
            latent_index = min(latent_index, cfg.num_train_frame - 1)
            ret.update({'wbounds': can_bounds, 'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index,
                        'frame_index': frame_index})
            # what prepare_inside_pts (:117-140) reads, for every training view in order
            nv = self.ims.shape[1]
            if train_item.image_steps(cfg) == 'device':    # get_mask (:102-115) stopped after decoding
                read = imread if imread is not None else _imread
                msks = [mask_item.read_cihp(self.data_root, self.ims[i, v], read) for v in range(nv)]
                H0, W0 = np.shape(msks[0])[:2]
                keys, ret['meta'] = mask_item.mask_fields(msks, [self.Ks[v] for v in range(nv)],
                                                          [self.Ds[v] for v in range(nv)], H0, W0, True, 5)
                ret.update(keys)
            else:
                ret['msks'] = np.stack([self.get_mask(i, v) for v in range(nv)]).astype(np.uint8)
            ret['Ks'] = np.asarray(self.Ks, dtype=np.float32).copy()
            ret['RT'] = np.concatenate([self.Rs, self.Ts], axis=2).astype(np.float32)
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
                              "'neuralbody_b200.lib.datasets.light_stage.multi_view_mesh_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
