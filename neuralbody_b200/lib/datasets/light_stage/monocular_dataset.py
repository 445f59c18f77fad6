"""Drop-in for the reference's People-Snapshot training dataset lib/datasets/light_stage/monocular_dataset.py (selected
through `train_dataset_module / train_dataset_path` and `test_dataset_module / test_dataset_path`, which name the same
file).

Split 'train': upstream's item carries N_rand rays that if_nerf_data_utils.sample_ray builds on the host (:106-107, float64
get_rays over the whole 1080 x 1080 image, three np.argwhere passes, the get_near_far rejection rounds).  This item runs
upstream's image steps unchanged (decode, undistort, INTER_AREA / INTER_NEAREST resize, background) and prepare_input, and
carries in place of the six ray keys the processed image `img` (H,W,3) float32, the pixel classes of sample_ray
`ray_class` (H,W) uint8, the camera `train_cam` (float32 K, float64 R and T, as upstream hands them to get_rays) and
`can_bounds`, with a host copy under `meta` (see multi_view_dataset.py, the ZJU-MoCap drop-in, for the keys).  Every
other key is upstream's, including `msk`, `K` and `RT`.  neuralbody_b200's renderers sample the rays on the GPU
(Renderer.train_rays).  Split 'test' carries the image and camera without the class map, and Renderer.camera_rays builds
the view's rays and colours on the GPU (nb_image_rays_f64 with the float32-K kind).
With `dataset_image_steps: 'device'` the item stops after decoding: it carries the decoded uint8 image and mask, K and D
(train_item.device_fields) in place of the processed image and class map, and the renderer runs the undistort, resize,
background and class map on the GPU (Renderer.item_images, nb_item_images).

`make_dataset_class(base)` builds the subclass over any base with the reference's attributes (`data_root`, `split`, `cam`,
`params`, `nrays`, `prepare_input`); `Dataset` is the one over the reference's own Dataset, resolved on first use.  OpenCV
and imageio are imported only when an item is built.  The module name in the yaml must be this module's
(`neuralbody_b200.lib.datasets.light_stage.monocular_dataset`), not upstream's, which it loads."""
import importlib
import os

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import train_item
from neuralbody_b200.lib.datasets.light_stage.multi_view_dataset import _bound_2d_mask, _cv2, _imread

REFERENCE_MODULE = "lib.datasets.light_stage.monocular_dataset"


def make_dataset_class(base, cv2=None, imread=None, bound_2d_mask=None):
    """-> a subclass of `base` whose __getitem__ returns the image (and for split 'train' its pixel classes) in place of the
    rays.
    `cv2`, `imread`, `bound_2d_mask`: as multi_view_dataset.make_dataset_class."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            read = imread if imread is not None else _imread
            if train_item.image_steps(cfg) == 'device':
                return self._device_item(index, cfg, cv, read)
            # monocular_dataset.py:74-104
            img_path = os.path.join(self.data_root, 'image', '{}.jpg'.format(index))
            img = read(img_path).astype(np.float32) / 255.
            msk_path = os.path.join(self.data_root, 'mask', '{}.png'.format(index))
            msk = read(msk_path)
            frame_index = index
            K = self.cam['K']
            D = self.cam['D']
            img = cv.undistort(img, K, D)
            msk = cv.undistort(msk, K, D)
            R = self.cam['R']
            T = self.cam['T'][:, None]
            RT = np.concatenate([R, T], axis=1).astype(np.float32)
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(frame_index)
            H, W = int(img.shape[0] * cfg.ratio), int(img.shape[1] * cfg.ratio)
            img = cv.resize(img, (W, H), interpolation=cv.INTER_AREA)
            msk = cv.resize(msk, (W, H), interpolation=cv.INTER_NEAREST)
            if cfg.mask_bkgd:
                img[msk == 0] = 0
                if cfg.white_bkgd:
                    img[msk == 0] = 1
            K = K.copy().astype(np.float32)
            K[:2] = K[:2] * cfg.ratio
            # what sample_ray (:106-107) reads
            ret = {'coord': coord, 'out_sh': out_sh, 'msk': msk}
            if self.split == 'train':
                bm = (bound_2d_mask or _bound_2d_mask)(can_bounds, K, np.concatenate([R, T], axis=1), H, W)
                ret.update(train_item.train_fields(img, train_item.class_map_snapshot(msk, bm), K, R, T, can_bounds, self.nrays,
                                                   cfg.body_sample_ratio, cfg.face_sample_ratio))
            else:
                ret.update(train_item.test_fields(img, K, R, T, can_bounds))
            return self._finish(ret, index, cv, Rh, Th, bounds, K, RT)

        def _device_item(self, index, cfg, cv, read):
            """`dataset_image_steps: 'device'`: the decoded image and mask and the camera in place of the processed image,
            class map and `msk` (train_item.device_fields; Renderer.item_images writes `msk` back); the rest as the host
            item."""
            img_u8 = np.asarray(read(os.path.join(self.data_root, 'image', '{}.jpg'.format(index))))
            msk_u8 = np.asarray(read(os.path.join(self.data_root, 'mask', '{}.png'.format(index))))
            K, D = self.cam['K'], self.cam['D']
            R = self.cam['R']
            T = self.cam['T'][:, None]
            RT = np.concatenate([R, T], axis=1).astype(np.float32)
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(index)
            H, W = int(img_u8.shape[0] * cfg.ratio), int(img_u8.shape[1] * cfg.ratio)
            Ks = K.copy().astype(np.float32)
            Ks[:2] = Ks[:2] * cfg.ratio
            train = self.split == 'train'
            bm = (bound_2d_mask or _bound_2d_mask)(can_bounds, Ks, np.concatenate([R, T], axis=1), H, W) if train else None
            ret, meta = train_item.device_fields(img_u8, msk_u8, K, D, H, W, cfg.mask_bkgd, cfg.white_bkgd, True,
                                                 train_item.CLASS_SNAPSHOT if train else None, bm)
            ret.update({'coord': coord, 'out_sh': out_sh})
            if train:
                ret.update(train_item.camera_fields(Ks, R, T, can_bounds, self.nrays, cfg.body_sample_ratio,
                                                    cfg.face_sample_ratio))
            else:
                ret.update(train_item.camera_fields(Ks, R, T, can_bounds))
            ret['meta'].update(meta)
            return self._finish(ret, index, cv, Rh, Th, bounds, Ks, RT)

        def _finish(self, ret, index, cv, Rh, Th, bounds, K, RT):
            # :121-136
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': index, 'frame_index': index,
                        'view_index': 0})
            Rh0 = self.params['pose'][index][:3]
            R0 = cv.Rodrigues(Rh0)[0].astype(np.float32)
            Th0 = self.params['trans'][index].astype(np.float32)
            ret.update({'R0_snap': R0, 'Th0_snap': Th0, 'K': K, 'RT': RT})
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
            raise ImportError("%s resolved to this drop-in: set train_dataset_module / test_dataset_module to "
                              "'neuralbody_b200.lib.datasets.light_stage.monocular_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset, imread=lambda p: ref.imageio.imread(p),
                                      bound_2d_mask=ref.if_nerf_dutils.get_bound_2d_mask)
    return _dataset
