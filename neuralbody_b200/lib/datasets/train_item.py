"""What the training dataset drop-ins (light_stage/multi_view_dataset.py, light_stage/monocular_dataset.py) put in an item
in place of upstream's rays: the image, the pixel classes upstream's sampler draws from (split 'train') and the camera the
GPU ray generators (neuralbody_b200.rays.train_rays through Renderer.train_rays; rays.dataset_image_rays through
Renderer.camera_rays for split 'test') read.  numpy only: this runs in data-loader workers,
which never touch CUDA."""
import numpy as np

BODY, FACE, BOUND = 1, 2, 4      # NB_TRAIN_CLASS_* (include/neuralbody_b200.h)
CLASS_H36M, CLASS_SNAPSHOT = 1, 2      # NB_ITEM_CLASS_*
RAY_KEYS = ('rgb', 'ray_o', 'ray_d', 'near', 'far', 'mask_at_box')


def class_map_h36m(msk, bound_mask):
    """sample_ray_h36m's lists (if_nerf_data_utils.py:160-190) as bits of one (H,W) uint8 map: body `msk * bound == 1`,
    face `== 13`, bound `bound_mask == 1` after the border pixels (msk 100) are taken out of it."""
    msk = msk * bound_mask
    bound_mask = bound_mask.copy()
    bound_mask[msk == 100] = 0
    return class_bits(msk == 1, msk == 13, bound_mask == 1)


def class_map_snapshot(msk, bound_mask):
    """sample_ray's lists (if_nerf_data_utils.py:79-108): body `msk * bound != 0`, face `== 13`, bound `bound_mask == 1`."""
    msk = msk * bound_mask
    return class_bits(msk != 0, msk == 13, bound_mask == 1)


def class_bits(body, face, bound):
    return (body * np.uint8(BODY) | face * np.uint8(FACE) | bound * np.uint8(BOUND)).astype(np.uint8)


def check_lists(class_map, n_rays, body_ratio, face_ratio):
    """Raise upstream's ValueError (np.random.randint(0, 0, n) with n > 0) where the first sampling round would: draws
    from an empty body or bound list."""
    n_body = int(n_rays * body_ratio)
    n_rand = n_rays - n_body - int(n_rays * face_ratio)
    if (n_body > 0 and not (class_map & BODY).any()) or (n_rand > 0 and not (class_map & BOUND).any()):
        raise ValueError("high <= 0")


def train_fields(img, class_map, K, R, T, can_bounds, n_rays, body_ratio, face_ratio):
    """The item keys that replace upstream's six ray keys, and the host copy under 'meta' the renderer reads."""
    check_lists(class_map, n_rays, body_ratio, face_ratio)
    ret = camera_fields(K, R, T, can_bounds, n_rays, body_ratio, face_ratio)
    ret.update({'img': np.ascontiguousarray(img, dtype=np.float32), 'ray_class': class_map})
    return ret


def test_fields(img, K, R, T, can_bounds):
    """Split 'test': the item keys that replace upstream's six (the whole view's box-hit rays and colours), and the host
    copy under 'meta' the renderer reads (Renderer.camera_rays)."""
    ret = camera_fields(K, R, T, can_bounds)
    ret['img'] = np.ascontiguousarray(img, dtype=np.float32)
    return ret


def camera_fields(K, R, T, can_bounds, n_rays=None, body_ratio=None, face_ratio=None):
    """The camera keys of either split (`train_cam`, `can_bounds` and their host copy under 'meta'); split 'train' (n_rays
    given) adds N_rand and the two sample ratios to 'meta'."""
    from neuralbody_b200.rays import train_camera
    kind, cam = train_camera(K, R, T, can_bounds)
    ret = {'train_cam': cam, 'can_bounds': can_bounds}
    ret['meta'] = {'train_cam': cam, 'train_k_kind': kind, 'can_bounds': can_bounds}
    if n_rays is not None:
        ret['meta'].update({'N_rand': int(n_rays), 'body_sample_ratio': float(body_ratio),
                            'face_sample_ratio': float(face_ratio)})
    return ret

def image_steps(cfg):
    """cfg.dataset_image_steps, 'host' when the config lacks the key (upstream's cfg under the reference process)."""
    steps = cfg.get('dataset_image_steps', 'host') if hasattr(cfg, 'get') else getattr(cfg, 'dataset_image_steps', 'host')
    if steps not in ('host', 'device'):
        raise ValueError("dataset_image_steps must be 'host' or 'device' (got %r)" % (steps,))
    return steps


def device_fields(img_u8, msk_u8, K, D, H, W, mask_bkgd, white_bkgd, keep_msk, class_rule=None, bound_mask=None):
    """`dataset_image_steps: 'device'`: the keys that replace the processed image (and class map, and for People-Snapshot
    `msk`), stopping after decoding.  img_u8 (H0,W0,3) and msk_u8 (H0,W0) uint8 as decoded, the camera K, D at that size,
    the output size (H, W); split 'train' adds the class rule (CLASS_H36M / CLASS_SNAPSHOT) and upstream's bound mask at
    (H, W).  Renderer.item_images turns a batch of these into `img`, `ray_class` and `msk` on the GPU (nb_item_images).
    Geometry the kernel does not implement raises ValueError: a resize other than a copy or an exact 2x reduction, a
    distortion model other than 4, 5 or 8 coefficients."""
    from neuralbody_b200 import images
    img_u8, msk_u8 = np.asarray(img_u8), np.asarray(msk_u8)
    if img_u8.dtype != np.uint8 or img_u8.ndim != 3 or img_u8.shape[2] != 3 or msk_u8.dtype != np.uint8 \
            or msk_u8.shape != img_u8.shape[:2]:
        raise ValueError("the device image steps take a (H0,W0,3) uint8 image and its (H0,W0) uint8 mask (got %s %s, %s %s)"
                         % (img_u8.dtype, img_u8.shape, msk_u8.dtype, msk_u8.shape))
    if img_u8.shape[1] > images.capi.NB_ITEM_MAX_W:
        raise ValueError("the device image steps take images up to %d pixels wide" % images.capi.NB_ITEM_MAX_W)
    images.reduction(img_u8.shape[0], img_u8.shape[1], H, W)
    n_dist, cam = images.item_camera(K, D)
    ret = {'img_u8': np.ascontiguousarray(img_u8), 'msk_u8': np.ascontiguousarray(msk_u8)}
    meta = {'image_cam': cam, 'image_n_dist': n_dist, 'image_size': np.array([H, W], np.int64),
            'image_bkgd': (2 if white_bkgd else 1) if mask_bkgd else 0, 'image_class': 0, 'image_msk': int(bool(keep_msk))}
    if class_rule is not None:
        bound_mask = np.asarray(bound_mask)
        if bound_mask.shape != (H, W):
            raise ValueError("the bound mask must be (H, W) = (%d, %d) (got %s)" % (H, W, bound_mask.shape))
        ret['bound_mask'] = np.ascontiguousarray(bound_mask, dtype=np.uint8)
        meta['image_class'] = int(class_rule)
    return ret, meta
