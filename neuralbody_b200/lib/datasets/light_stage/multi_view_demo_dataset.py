"""Drop-in for the reference's novel-view dataset lib/datasets/light_stage/multi_view_demo_dataset.py (selected through
`test_dataset_module / test_dataset_path` in `novel_view_cfg`, for `run.py --type visualize` with `vis_novel_view True`).

Upstream's item carries the view's rays, built on the host by render_utils.image_rays for every view (:151-152: numpy
get_rays + get_near_far over the whole image, then the mask_at_box compaction, ~8 MB of rays for a 512 x 512 view). This
item carries the render camera instead, under new keys (`RT` / `Ks` already name the mask views): `cam_RT` =
render_w2c[index] (4,4) and `cam_K` = the dataset's K (3,3), in the dtype upstream hands them to image_rays (float64
with ZJU-MoCap's annotations), and `can_bounds` (2,3) float32. neuralbody_b200's renderers generate the same rays, near,
far and mask_at_box from them on the GPU (Renderer.camera_rays). `meta` holds the same three arrays: upstream's
visualize loop (run.py) moves every key but `meta` to the GPU, so the renderer reads the camera there with no copy back
to the host. Every other key is upstream's: coord, out_sh, bounds, R, Th, latent_index, frame_index, view_index and the
mask views msks / Ks / RT from upstream's own get_mask (decoded, undistorted and dilated on the host) and INTER_NEAREST
resize. Every view renders the same frame (cfg.ith_frame), so its masks are built once and kept by the dataset.

With `dataset_image_steps: 'device'` (default 'host') the item stops after decoding the masks: it ships `msks_u8`
(nv,H0,W0) uint8 as read, before upstream's binarisation, in place of `msks`, and each view's camera (upstream's
`Ks[nv]` with rows 0-1 divided by cfg.ratio, `Ds[nv]`) and the recipe (binarise, 5 x 5 dilation, the resize to
cfg.H * ratio x cfg.W * ratio) under `meta` (lib/datasets/mask_item.py).  The `_mmsk` renderer builds the same `msks` on
the GPU (Renderer.mask_views, nb_mask_views).

`Dataset` subclasses the reference's own Dataset, resolved when it is first asked for (so this module imports without the
reference tree); `make_dataset_class(base)` builds the same subclass over any base with the reference's attributes
(`K`, `Ks`, `RT`, `render_w2c`, `prepare_input`, `get_mask`, and for the 'device' items `data_root`, `ims`, `Ds`).  OpenCV is imported only when an item is built.  The module
name in `test_dataset_module` must be this module's (`neuralbody_b200.lib.datasets.light_stage.multi_view_demo_dataset`),
not upstream's, which it loads."""
import importlib

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import mask_item, train_item

REFERENCE_MODULE = "lib.datasets.light_stage.multi_view_demo_dataset"


def _cv2():
    import cv2
    return cv2


def resized_masks(cv, msks, H, W):
    """multi_view_demo_dataset.py:143-148 (and the perform set's :138-143): each view to (W, H), INTER_NEAREST."""
    return np.array([cv.resize(m, (W, H), interpolation=cv.INTER_NEAREST) for m in msks])


def _imread(path):
    import imageio
    return imageio.imread(path)


def decoded_masks(ds, i, H, W, imread):
    """`dataset_image_steps: 'device'`: upstream's get_mask(i) (multi_view_demo_dataset.py:107-129, the perform set's
    :105-127) stopped after decoding -> (the item keys, the 'meta' keys) of mask_item.mask_fields."""
    cfg = get_active_cfg()
    msks, Ks = [], []
    for nv, im in enumerate(ds.ims[i]):
        msks.append(mask_item.read_cihp(ds.data_root, im, imread))
        K = ds.Ks[nv].copy()
        K[:2] = K[:2] / cfg.ratio
        Ks.append(K)
    return mask_item.mask_fields(msks, Ks, [ds.Ds[nv] for nv in range(len(msks))], H, W, True, 5)


def make_dataset_class(base, cv2=None, imread=None):
    """-> a subclass of `base` whose __getitem__ returns the render camera in place of the rays.  `cv2`: the module
    providing resize, INTER_NEAREST and Rodrigues (OpenCV, imported on first use, when None); `imread`: the mask reader of
    the 'device' items (imageio.imread, as upstream, when None)."""

    class Dataset(base):
        def _frame_masks(self, i, H, W):
            cache = self.__dict__.setdefault("_nb_masks", {})
            if (i, H, W) not in cache:
                cache.clear()
                cache[(i, H, W)] = resized_masks(cv2 if cv2 is not None else _cv2(), self.get_mask(i), H, W)
            return cache[(i, H, W)]

        def _frame_decoded(self, i, H, W):
            cache = self.__dict__.setdefault("_nb_decoded", {})
            if (i, H, W) not in cache:
                cache.clear()
                cache[(i, H, W)] = decoded_masks(self, i, H, W, imread if imread is not None else _imread)
            return cache[(i, H, W)]

        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            # multi_view_demo_dataset.py:132-149
            i = cfg.ith_frame
            latent_index = i
            frame_index = i + cfg.begin_ith_frame
            view_index = index
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(frame_index)
            H, W = int(cfg.H * cfg.ratio), int(cfg.W * cfg.ratio)
            device = train_item.image_steps(cfg) == 'device'
            msks, mask_meta = self._frame_decoded(i, H, W) if device else ({'msks': self._frame_masks(i, H, W)}, {})
            ret = {'coord': coord, 'out_sh': out_sh}
            # :164-177
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            latent_index = min(latent_index, cfg.num_train_frame - 1)
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index, 'frame_index': frame_index,
                        'view_index': view_index})
            ret.update(msks)
            ret.update({'Ks': self.Ks, 'RT': self.RT})
            # what image_rays (:151-152) reads
            ret.update({'cam_RT': self.render_w2c[index], 'cam_K': self.K, 'can_bounds': can_bounds})
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
                              "'neuralbody_b200.lib.datasets.light_stage.multi_view_demo_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset)
    return _dataset
