"""Drop-in for the reference's ZJU-MoCap training dataset lib/datasets/light_stage/multi_view_dataset.py (selected through
`train_dataset_module / train_dataset_path` and `test_dataset_module / test_dataset_path`, which name the same file).

Split 'train': upstream's item carries N_rand rays that if_nerf_data_utils.sample_ray_h36m builds on the host (:154-155:
float64 get_rays over the whole image, three np.argwhere passes, then the get_near_far rejection rounds).  This item runs
upstream's image steps unchanged (decode, resize, get_mask, undistort, INTER_AREA / INTER_NEAREST resize, background) and
prepare_input, and carries in place of the six ray keys (rgb, ray_o, ray_d, near, far, mask_at_box):
  - `img` (H,W,3) float32: the processed image upstream samples rgb from;
  - `ray_class` (H,W) uint8: the body / face / bound pixel classes of sample_ray_h36m, from upstream's own
    get_bound_2d_mask and mask arithmetic (neuralbody_b200.lib.datasets.train_item);
  - `train_cam` (30,) float64: inv(K), R, T, the camera centre and can_bounds (neuralbody_b200.rays.train_camera), and
    `can_bounds` (2,3) float32;
  - `meta`: a host copy of the camera with N_rand and the two sample ratios.  Upstream's trainer moves every key but
    'meta' to the GPU, so the renderer reads it with no copy back.
neuralbody_b200's renderers draw the pixels and build the rays, near, far and rgb on the GPU (Renderer.train_rays) and
write upstream's six keys into the batch, so the trainer and the evaluator run unchanged.  Where upstream's
np.random.randint would raise (an empty body or bound list) the item raises the same ValueError.  Split 'test' (the
evaluation views, whose upstream item carries every box-hit ray of the view and its colour) carries `img`, `train_cam`,
`can_bounds` and `meta` without the class map; Renderer.camera_rays builds the rays, near, far, rgb and mask_at_box on
the GPU (nb_image_rays_f64 with the image).
With `dataset_image_steps: 'device'` the item stops after decoding: it carries the decoded uint8 image and mask, K and D
(train_item.device_fields) in place of the processed image and class map, and the renderer runs the undistort, resize,
background and class map on the GPU (Renderer.item_images, nb_item_images).

`Dataset` subclasses the reference's own Dataset, resolved when it is first asked for; `make_dataset_class(base)` builds
the same subclass over any base with the reference's attributes (`data_root`, `human`, `split`, `ims`, `cam_inds`,
`cams`, `nrays`, `get_mask`, `prepare_input`).  OpenCV and imageio are imported only when an item is built.  The module
name in the yaml must be this module's (`neuralbody_b200.lib.datasets.light_stage.multi_view_dataset`), not upstream's,
which it loads."""
import importlib
import os

import numpy as np

from neuralbody_b200.lib.config import get_active_cfg
from neuralbody_b200.lib.datasets import train_item

REFERENCE_MODULE = "lib.datasets.light_stage.multi_view_dataset"


def _cv2():
    import cv2
    return cv2


def _imread(path):
    import imageio
    return imageio.imread(path)


def _bound_2d_mask(*args):
    from lib.utils.if_nerf import if_nerf_data_utils
    return if_nerf_data_utils.get_bound_2d_mask(*args)


def _frame(human, img_path):
    """multi_view_dataset.py:159-165: (frame_index, the index prepare_input reads)."""
    if human in ['CoreView_313', 'CoreView_315']:
        i = int(os.path.basename(img_path).split('_')[4])
        return i - 1, i
    i = int(os.path.basename(img_path)[:-4])
    return i, i


def make_dataset_class(base, cv2=None, imread=None, bound_2d_mask=None):
    """-> a subclass of `base` whose __getitem__ returns the image (and for split 'train' its pixel classes) in place of the
    rays.
    `cv2`: the module providing resize, undistort, INTER_AREA, INTER_NEAREST (OpenCV when None); `imread`: the image reader
    (imageio.imread, as upstream, when None); `bound_2d_mask`: upstream's if_nerf_data_utils.get_bound_2d_mask when None."""

    class Dataset(base):
        def __getitem__(self, index):
            cfg = get_active_cfg()
            cv = cv2 if cv2 is not None else _cv2()
            read = imread if imread is not None else _imread
            if train_item.image_steps(cfg) == 'device':
                return self._device_item(index, cfg, cv, read)
            # multi_view_dataset.py:121-152
            img_path = os.path.join(self.data_root, self.ims[index])
            img = read(img_path).astype(np.float32) / 255.
            img = cv.resize(img, (cfg.W, cfg.H))
            msk = self.get_mask(index)
            cam_ind = self.cam_inds[index]
            K = np.array(self.cams['K'][cam_ind])
            D = np.array(self.cams['D'][cam_ind])
            img = cv.undistort(img, K, D)
            msk = cv.undistort(msk, K, D)
            R = np.array(self.cams['R'][cam_ind])
            T = np.array(self.cams['T'][cam_ind]) / 1000.
            H, W = int(img.shape[0] * cfg.ratio), int(img.shape[1] * cfg.ratio)
            img = cv.resize(img, (W, H), interpolation=cv.INTER_AREA)
            msk = cv.resize(msk, (W, H), interpolation=cv.INTER_NEAREST)
            if cfg.mask_bkgd:
                img[msk == 0] = 0
                if cfg.white_bkgd:
                    img[msk == 0] = 1
            K[:2] = K[:2] * cfg.ratio
            frame_index, i = _frame(self.human, img_path)
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(i)
            # what sample_ray_h36m (:154-155) reads
            ret = {'coord': coord, 'out_sh': out_sh}
            if self.split == 'train':
                bm = (bound_2d_mask or _bound_2d_mask)(can_bounds, K, np.concatenate([R, T], axis=1), H, W)
                ret.update(train_item.train_fields(img, train_item.class_map_h36m(msk, bm), K, R, T, can_bounds, self.nrays,
                                                   cfg.body_sample_ratio, cfg.face_sample_ratio))
            else:
                ret.update(train_item.test_fields(img, K, R, T, can_bounds))
            return self._finish(ret, cfg, cv, Rh, Th, bounds, frame_index, cam_ind)

        def _device_item(self, index, cfg, cv, read):
            """`dataset_image_steps: 'device'`: the decoded image, upstream's get_mask and the camera in place of the
            processed image and class map (train_item.device_fields); the rest as the host item."""
            img_path = os.path.join(self.data_root, self.ims[index])
            img_u8 = np.asarray(read(img_path))
            if img_u8.shape[:2] != (cfg.H, cfg.W):
                raise ValueError("the device image steps need the image at (cfg.H, cfg.W) = (%d, %d), where upstream's "
                                 "first resize is a copy (got %s)" % (cfg.H, cfg.W, img_u8.shape[:2]))
            msk = self.get_mask(index)
            cam_ind = self.cam_inds[index]
            K = np.array(self.cams['K'][cam_ind])
            D = np.array(self.cams['D'][cam_ind])
            R = np.array(self.cams['R'][cam_ind])
            T = np.array(self.cams['T'][cam_ind]) / 1000.
            H, W = int(img_u8.shape[0] * cfg.ratio), int(img_u8.shape[1] * cfg.ratio)
            train = self.split == 'train'
            Ks = K.copy()
            Ks[:2] = Ks[:2] * cfg.ratio
            frame_index, i = _frame(self.human, img_path)
            coord, out_sh, can_bounds, bounds, Rh, Th = self.prepare_input(i)
            bm = (bound_2d_mask or _bound_2d_mask)(can_bounds, Ks, np.concatenate([R, T], axis=1), H, W) if train else None
            ret, meta = train_item.device_fields(img_u8, msk, K, D, H, W, cfg.mask_bkgd, cfg.white_bkgd, False,
                                                 train_item.CLASS_H36M if train else None, bm)
            ret.update({'coord': coord, 'out_sh': out_sh})
            if train:
                ret.update(train_item.camera_fields(Ks, R, T, can_bounds, self.nrays, cfg.body_sample_ratio,
                                                    cfg.face_sample_ratio))
            else:
                ret.update(train_item.camera_fields(Ks, R, T, can_bounds))
            ret['meta'].update(meta)
            return self._finish(ret, cfg, cv, Rh, Th, bounds, frame_index, cam_ind)

        def _finish(self, ret, cfg, cv, Rh, Th, bounds, frame_index, cam_ind):
            # :168-180
            R = cv.Rodrigues(Rh)[0].astype(np.float32)
            latent_index = (frame_index - cfg.begin_ith_frame) // cfg.frame_interval
            if cfg.test_novel_pose:
                latent_index = cfg.num_train_frame - 1
            ret.update({'bounds': bounds, 'R': R, 'Th': Th, 'latent_index': latent_index, 'frame_index': frame_index,
                        'cam_ind': cam_ind})
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
                              "'neuralbody_b200.lib.datasets.light_stage.multi_view_dataset'" % REFERENCE_MODULE)
        _dataset = make_dataset_class(ref.Dataset, imread=lambda p: ref.imageio.imread(p),
                                      bound_2d_mask=ref.if_nerf_dutils.get_bound_2d_mask)
    return _dataset
