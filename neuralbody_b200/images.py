"""The training datasets' image steps after decoding on the device (nb_item_images): undistort, the resize by cfg.ratio
(a copy or an exact 2x reduction), the background and the sampler's class map, bit for bit with OpenCV's host steps
(oracle/item_images.py restates them).  Items of the `dataset_image_steps: 'device'` kind carry the decoded image and
mask and the camera; Renderer.item_images runs this on a collated batch.

`mask_views` is the demo and mesh datasets' counterpart for their mask views (nb_mask_views): the optional binarisation,
the undistort, the optional 5 x 5 dilation and the INTER_NEAREST resize, per view with its own camera;
Renderer.mask_views runs it on a collated batch."""
import ctypes as C

import numpy as np
import torch

from . import capi

BKGD = {"none": capi.NB_ITEM_BKGD_NONE, "black": capi.NB_ITEM_BKGD_BLACK, "white": capi.NB_ITEM_BKGD_WHITE}


def item_camera(K, D):
    """K (3,3) and D (4, 5 or 8 coefficients) at the decoded size, in any float dtype -> (n_dist, (NB_ITEM_CAM_DOUBLES,)
    float64): K row-major, then D zero-padded to 8, each value exact (float32 -> float64 is)."""
    K = np.asarray(K)
    D = np.asarray(D)
    if K.shape != (3, 3) or K.dtype not in (np.float32, np.float64) or D.dtype not in (np.float32, np.float64):
        raise ValueError("K must be a float32 or float64 (3,3) and D float32 or float64 (got %s %s, %s)"
                         % (K.dtype, K.shape, D.dtype))
    if D.size not in (4, 5, 8) or D.size != max(D.shape, default=0):
        raise ValueError("D must be a vector of 4, 5 or 8 distortion coefficients (got shape %s)" % (D.shape,))
    cam = np.zeros(capi.NB_ITEM_CAM_DOUBLES)
    cam[:9] = K.astype(np.float64).ravel()
    cam[9:9 + D.size] = D.astype(np.float64).ravel()
    return D.size, cam


def reduction(H0, W0, H, W):
    """1 when the item's steps keep the decoded size, 2 for an exact 2x reduction; ValueError for any other geometry (the
    kernel implements only these two: INTER_AREA's fast path and a copy)."""
    if (H, W) == (H0, W0):
        return 1
    if (2 * H, 2 * W) == (H0, W0):
        return 2
    raise ValueError("the device image steps resize only by a copy or an exact 2x reduction (got %dx%d -> %dx%d)"
                     % (H0, W0, H, W))


def item_images(img_u8, msk_u8, cams, n_dist, H, W, bkgd=capi.NB_ITEM_BKGD_NONE, class_rule=capi.NB_ITEM_CLASS_NONE,
                bound=None):
    """nb_item_images on a batch: img_u8 (B,H0,W0,3) and msk_u8 (B,H0,W0) uint8 CUDA tensors on one device, cams
    (B, NB_ITEM_CAM_DOUBLES) float64 on the host (stacked `item_camera` results, all with `n_dist` coefficients), the
    output size, the background (NB_ITEM_BKGD_*) and the class rule (NB_ITEM_CLASS_*) with its (B,H,W) uint8 bound mask.
    Nothing synchronises with the host.  -> img (B,H,W,3) float32, msk (B,H,W) uint8, class map (B,H,W) uint8 or None."""
    lib = capi.load()
    if not (torch.is_tensor(img_u8) and torch.is_tensor(msk_u8)) or img_u8.device.type != "cuda":
        raise ValueError("img_u8 and msk_u8 must be CUDA tensors")
    dev = img_u8.device
    B, H0, W0 = (int(s) for s in msk_u8.shape)
    if tuple(img_u8.shape) != (B, H0, W0, 3) or img_u8.dtype != torch.uint8 or msk_u8.dtype != torch.uint8 \
            or msk_u8.device != dev:
        raise ValueError("img_u8 must be (B,H0,W0,3) and msk_u8 (B,H0,W0), uint8 on one device (got %s %s, %s %s)"
                         % (tuple(img_u8.shape), img_u8.dtype, tuple(msk_u8.shape), msk_u8.dtype))
    reduction(H0, W0, H, W)
    cams = np.ascontiguousarray(cams, dtype=np.float64)
    if cams.shape != (B, capi.NB_ITEM_CAM_DOUBLES):
        raise ValueError("cams must be (B, %d) (got %s)" % (capi.NB_ITEM_CAM_DOUBLES, cams.shape))
    rule = int(class_rule) != capi.NB_ITEM_CLASS_NONE
    if rule != (bound is not None):
        raise ValueError("a class rule needs the bound mask, and only a class rule takes one")
    with torch.cuda.device(dev):
        a = capi.nb_item_images_args()
        a.B, a.H0, a.W0, a.H, a.W = B, H0, W0, int(H), int(W)
        a.n_dist, a.bkgd, a.class_rule = int(n_dist), int(bkgd), int(class_rule)
        img_u8, msk_u8 = img_u8.contiguous(), msk_u8.contiguous()
        a.img_u8, a.msk_u8 = img_u8.data_ptr(), msk_u8.data_ptr()
        cams_dev = torch.from_numpy(cams).pin_memory().to(dev, non_blocking=True)
        a.cams = cams_dev.data_ptr()
        img = torch.empty((B, int(H), int(W), 3), dtype=torch.float32, device=dev)
        msk = torch.empty((B, int(H), int(W)), dtype=torch.uint8, device=dev)
        a.img, a.msk = img.data_ptr(), msk.data_ptr()
        cmap = None
        if rule:
            bound = bound.to(dev).contiguous()
            if tuple(bound.shape) != (B, int(H), int(W)) or bound.dtype != torch.uint8:
                raise ValueError("bound must be (B,H,W) uint8 (got %s %s)" % (tuple(bound.shape), bound.dtype))
            cmap = torch.empty((B, int(H), int(W)), dtype=torch.uint8, device=dev)
            a.bound, a.class_map = bound.data_ptr(), cmap.data_ptr()
        capi.check(lib.nb_item_images(C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "nb_item_images")
        return img, msk, cmap


def mask_views(msk_u8, cams, n_dist, H, W, binarise, dilate):
    """nb_mask_views on one item's views: msk_u8 (nv,H0,W0) uint8 CUDA tensor as decoded, cams (nv, NB_ITEM_CAM_DOUBLES)
    float64 on the host (stacked `item_camera` results; `n_dist` the largest of their coefficient counts: the rest are
    zero), the output size (a copy or an exact 2x reduction, see `reduction`), `binarise` (undistort m != 0) and `dilate`
    (0 or 5).  Everything is validated before the launch; nothing synchronises with the host.  -> msks (nv,H,W) uint8."""
    lib = capi.load()
    if not torch.is_tensor(msk_u8) or msk_u8.device.type != "cuda":
        raise ValueError("msk_u8 must be a CUDA tensor")
    if msk_u8.dim() != 3 or msk_u8.dtype != torch.uint8:
        raise ValueError("msk_u8 must be (nv,H0,W0) uint8 (got %s %s)" % (tuple(msk_u8.shape), msk_u8.dtype))
    dev = msk_u8.device
    nv, H0, W0 = (int(s) for s in msk_u8.shape)
    if nv < 1 or W0 > capi.NB_ITEM_MAX_W:
        raise ValueError("mask_views takes at least one view up to %d pixels wide (got %d views of %dx%d)"
                         % (capi.NB_ITEM_MAX_W, nv, H0, W0))
    reduction(H0, W0, H, W)
    cams = np.ascontiguousarray(cams, dtype=np.float64)
    if cams.shape != (nv, capi.NB_ITEM_CAM_DOUBLES):
        raise ValueError("cams must be (nv, %d) (got %s)" % (capi.NB_ITEM_CAM_DOUBLES, cams.shape))
    if int(n_dist) not in (4, 5, 8) or int(dilate) not in (0, 5) or int(binarise) not in (0, 1):
        raise ValueError("n_dist must be 4, 5 or 8, dilate 0 or 5 and binarise 0 or 1 (got %s, %s, %s)"
                         % (n_dist, dilate, binarise))
    with torch.cuda.device(dev):
        a = capi.nb_mask_views_args()
        a.nv, a.H0, a.W0, a.H, a.W = nv, H0, W0, int(H), int(W)
        a.n_dist, a.binarise, a.dilate = int(n_dist), int(binarise), int(dilate)
        msk_u8 = msk_u8.contiguous()
        a.msk_u8 = msk_u8.data_ptr()
        cams_dev = torch.from_numpy(cams).pin_memory().to(dev, non_blocking=True)
        a.cams = cams_dev.data_ptr()
        ws = None
        if a.dilate:
            a.workspace_bytes = lib.nb_mask_views_workspace_bytes(nv, H0, W0)
            ws = torch.empty(a.workspace_bytes, dtype=torch.uint8, device=dev)
            a.workspace = ws.data_ptr()
        out = torch.empty((nv, int(H), int(W)), dtype=torch.uint8, device=dev)
        a.msks = out.data_ptr()
        capi.check(lib.nb_mask_views(C.byref(a), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "nb_mask_views")
        return out
