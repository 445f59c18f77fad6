"""What the demo and mesh dataset drop-ins (light_stage/multi_view_demo_dataset.py, multi_view_perform_dataset.py,
monocular_demo_dataset.py, multi_view_mesh_dataset.py, monocular_mesh_dataset.py) put in an item in place of upstream's
processed mask views under `dataset_image_steps: 'device'`: the decoded masks and, under 'meta', each view's camera and
the recipe.  Renderer.mask_views turns a batch of these into upstream's `msks` (or `msk`) on the GPU (nb_mask_views, bit
for bit with upstream's host steps).  numpy only: this runs in data-loader workers, which never touch CUDA."""
import os

import numpy as np


def read_cihp(data_root, im, imread):
    """The decoded ZJU-MoCap part mask of image `im` (mask_cihp/<im>.png), as upstream's get_mask reads it."""
    return imread(os.path.join(data_root, 'mask_cihp', im)[:-4] + '.png')


def mask_fields(msks_u8, Ks, Ds, H, W, binarise, dilate):
    """-> (the item keys, the 'meta' keys) of `nv` decoded mask views: msks_u8 a sequence of (H0,W0) uint8 arrays as
    decoded, Ks (3,3) and Ds (4, 5 or 8 coefficients) each view's camera at that size, the output size (H, W), `binarise`
    (upstream's (m != 0) before the undistort) and `dilate` (0, or 5 for upstream's 5 x 5 cv2.dilate).  The item ships
    `msks_u8` (nv,H0,W0) uint8; meta holds `mask_cams` (nv, NB_ITEM_CAM_DOUBLES) float64, `mask_n_dist`, `mask_size` (2,)
    int64, `mask_binarise` and `mask_dilate`.  Geometry the kernel does not implement raises ValueError here, before any GPU
    work: a mask that is not 2-D uint8, views of different sizes, a resize other than a copy or an exact 2x reduction, a
    distortion model other than 4, 5 or 8 coefficients, an image wider than NB_ITEM_MAX_W."""
    from neuralbody_b200 import images
    msks = [np.asarray(m) for m in msks_u8]
    if not msks or any(m.dtype != np.uint8 or m.ndim != 2 for m in msks):
        raise ValueError("the device mask steps take 2-D uint8 masks as decoded (got %s)"
                         % [(m.dtype, m.shape) for m in msks])
    H0, W0 = msks[0].shape
    if any(m.shape != (H0, W0) for m in msks):
        raise ValueError("the mask views must share one size (got %s)" % [m.shape for m in msks])
    if W0 > images.capi.NB_ITEM_MAX_W:
        raise ValueError("the device mask steps take masks up to %d pixels wide (got %d)" % (images.capi.NB_ITEM_MAX_W, W0))
    images.reduction(H0, W0, H, W)
    if len(Ks) != len(msks) or len(Ds) != len(msks):
        raise ValueError("one camera per mask view (got %d views, %d K, %d D)" % (len(msks), len(Ks), len(Ds)))
    cams = [images.item_camera(K, D) for K, D in zip(Ks, Ds)]
    ret = {'msks_u8': np.ascontiguousarray(np.stack(msks))}
    meta = {'mask_cams': np.stack([c for _, c in cams]), 'mask_n_dist': max(n for n, _ in cams),
            'mask_size': np.array([H, W], np.int64), 'mask_binarise': int(bool(binarise)), 'mask_dilate': int(dilate)}
    return ret, meta
