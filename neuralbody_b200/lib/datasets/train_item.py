"""What the training dataset drop-ins (light_stage/multi_view_dataset.py, light_stage/monocular_dataset.py) put in an item
in place of upstream's rays: the image, the pixel classes upstream's sampler draws from (split 'train') and the camera the
GPU ray generators (neuralbody_b200.rays.train_rays through Renderer.train_rays; rays.dataset_image_rays through
Renderer.camera_rays for split 'test') read.  numpy only: this runs in data-loader workers,
which never touch CUDA."""
import numpy as np

BODY, FACE, BOUND = 1, 2, 4      # NB_TRAIN_CLASS_* (include/neuralbody_b200.h)
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
    from neuralbody_b200.rays import train_camera
    check_lists(class_map, n_rays, body_ratio, face_ratio)
    kind, cam = train_camera(K, R, T, can_bounds)
    ret = {'img': np.ascontiguousarray(img, dtype=np.float32), 'ray_class': class_map, 'train_cam': cam,
           'can_bounds': can_bounds}
    ret['meta'] = {'train_cam': cam, 'train_k_kind': kind, 'can_bounds': can_bounds, 'N_rand': int(n_rays),
                   'body_sample_ratio': float(body_ratio), 'face_sample_ratio': float(face_ratio)}
    return ret


def test_fields(img, K, R, T, can_bounds):
    """Split 'test': the item keys that replace upstream's six (the whole view's box-hit rays and colours), and the host
    copy under 'meta' the renderer reads (Renderer.camera_rays)."""
    from neuralbody_b200.rays import train_camera
    kind, cam = train_camera(K, R, T, can_bounds)
    ret = {'img': np.ascontiguousarray(img, dtype=np.float32), 'train_cam': cam, 'can_bounds': can_bounds}
    ret['meta'] = {'train_cam': cam, 'train_k_kind': kind, 'can_bounds': can_bounds}
    return ret
