"""numpy restatement of the reference's per-view evaluator (lib/evaluators/if_nerf.py, Evaluator.evaluate and
ssim_metric) for nb_eval_image and the evaluator drop-in.

`compare_ssim` restates scikit-image 0.14.2's skimage.measure.compare_ssim (the reference's requirements.txt pin) for the
arguments the evaluator passes, over scipy.ndimage.uniform_filter, the function skimage calls.  scikit-image itself is
not a dependency here: tests/test_eval_metrics_cpu.py pins the restatement against `ssim_bruteforce`, an independent
float64 definition with explicit 7 x 7 windows and reflect indexing.  Its parity to skimage itself is not pinned.

`evaluate_view` follows Evaluator.evaluate line by line (the scatter, the float32 MSE, PSNR, the box, the crop, SSIM) and
returns the crops' uint8 BGR bytes (`to_u8`, cv2's saturate_cast of the float64 image times 255).  With `png_dir` it also
crops with cv2.boundingRect and writes the PNGs from the float64 images as upstream does."""
import os

import numpy as np

WIN = 7


def uniform_filter(x):
    from scipy.ndimage import uniform_filter as uf
    return uf(x, size=WIN)


def compare_ssim(X, Y, win_size=None, gradient=False, data_range=None, multichannel=False, gaussian_weights=False,
                 full=False, **kwargs):
    """skimage.measure.compare_ssim of scikit-image 0.14.2 for the uniform-window, sample-covariance, mean-only case
    (the evaluator's `compare_ssim(img_pred, img_gt, multichannel=True)`)."""
    if gradient or gaussian_weights or full:
        raise NotImplementedError("the restatement covers the mean SSIM with the uniform window")
    if X.shape != Y.shape:
        raise ValueError("Input images must have the same dimensions.")
    if multichannel:
        args = dict(win_size=win_size, data_range=data_range)
        args.update(kwargs)
        nch = X.shape[-1]
        mssim = np.empty(nch)
        for ch in range(nch):
            mssim[..., ch] = compare_ssim(X[..., ch], Y[..., ch], **args)
        return mssim.mean()
    K1 = kwargs.pop('K1', 0.01)
    K2 = kwargs.pop('K2', 0.03)
    if kwargs.pop('use_sample_covariance', True) is not True:
        raise NotImplementedError("the restatement covers the sample covariance")
    if win_size is None:
        win_size = WIN
    if win_size != WIN:
        raise NotImplementedError("the restatement covers the 7 x 7 window")
    if np.any((np.asarray(X.shape) - win_size) < 0):
        raise ValueError("win_size exceeds image extent.  If the input is a multichannel (color) image, set "
                         "multichannel=True.")
    if data_range is None:
        if not np.issubdtype(X.dtype, np.floating):
            raise NotImplementedError("the restatement covers float images (dtype_range (-1, 1))")
        data_range = 2.0
    X = X.astype(np.float64)
    Y = Y.astype(np.float64)
    NP = win_size ** X.ndim
    cov_norm = NP / (NP - 1)
    ux = uniform_filter(X)
    uy = uniform_filter(Y)
    uxx = uniform_filter(X * X)
    uyy = uniform_filter(Y * Y)
    uxy = uniform_filter(X * Y)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    R = data_range
    C1 = (K1 * R) ** 2
    C2 = (K2 * R) ** 2
    A1, A2, B1, B2 = ((2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2))
    S = (A1 * A2) / (B1 * B2)
    pad = (win_size - 1) // 2
    return S[pad:-pad, pad:-pad].mean()


def ssim_bruteforce(X, Y):
    """The mean SSIM of two (h, w, c) images by its definition, independently of scipy: per channel, every pixel's 7 x 7
    window taken explicitly from the image padded by reflection (index -1 -> 0, -2 -> 1, h -> h-1), its sample means,
    variances and covariance, then S over the pixels 3 away from every edge, averaged, then the channels averaged."""
    X = np.asarray(X, np.float64)
    Y = np.asarray(Y, np.float64)
    h, w = X.shape[:2]
    if h < WIN or w < WIN:
        raise ValueError("win_size exceeds image extent")
    p = WIN // 2
    C1, C2 = (0.01 * 2) ** 2, (0.03 * 2) ** 2
    vals = []
    for ch in range(X.shape[2]):
        xs = np.pad(X[..., ch], p, mode="symmetric")
        ys = np.pad(Y[..., ch], p, mode="symmetric")
        wx = np.lib.stride_tricks.sliding_window_view(xs, (WIN, WIN)).reshape(h, w, WIN * WIN)
        wy = np.lib.stride_tricks.sliding_window_view(ys, (WIN, WIN)).reshape(h, w, WIN * WIN)
        mx, my = wx.mean(-1), wy.mean(-1)
        vx = ((wx - mx[..., None]) ** 2).sum(-1) / (WIN * WIN - 1)
        vy = ((wy - my[..., None]) ** 2).sum(-1) / (WIN * WIN - 1)
        vxy = ((wx - mx[..., None]) * (wy - my[..., None])).sum(-1) / (WIN * WIN - 1)
        S = (2 * mx * my + C1) * (2 * vxy + C2) / ((mx ** 2 + my ** 2 + C1) * (vx + vy + C2))
        vals.append(S[p:-p, p:-p].mean())
    return float(np.mean(vals))


def bounding_rect(mask):
    """cv2.boundingRect of a 2-D mask: (x, y, w, h) of its nonzero pixels, (0, 0, 0, 0) when there are none."""
    ys, xs = np.nonzero(mask)
    if ys.size == 0:
        return (0, 0, 0, 0)
    return (int(xs.min()), int(ys.min()), int(xs.max() - xs.min() + 1), int(ys.max() - ys.min() + 1))


def to_u8(img):
    """What cv2.imwrite stores for a float64 image: saturate_cast<uchar>, i.e. cvRound (round half to even; NaN or
    outside int32 -> INT_MIN) clamped to [0, 255]."""
    r = np.rint(np.asarray(img, np.float64))
    ok = (r >= -2147483648.0) & (r <= 2147483647.0)
    i = np.where(ok, r, -2147483648.0)
    return np.clip(i, 0, 255).astype(np.uint8)


def evaluate_view(rgb_pred, rgb_gt, mask_at_box, H, W, white_bkgd=False, eval_whole_img=False, png_dir=None,
                  frame_index=0, view_index=0):
    """Evaluator.evaluate on one view: rgb_pred, rgb_gt (n,3) float32, mask_at_box (H*W) -> dict with upstream's mse
    (float32, or float64 with eval_whole_img), psnr and ssim, the box (x, y, w, h) the crop takes (the whole image with
    eval_whole_img), the crops as uint8 BGR (crop_pred, crop_gt) and `mse_f64`, the same terms summed exactly in float64
    (math.fsum) over their count.  Raises upstream's ValueError for a count mismatch or a crop under 7 pixels."""
    import math
    rgb_pred = np.asarray(rgb_pred)
    rgb_gt = np.asarray(rgb_gt)
    mask = np.asarray(mask_at_box).reshape(H, W).astype(bool)
    white_bkgd = int(white_bkgd)
    img_pred = np.zeros((H, W, 3)) + white_bkgd
    img_pred[mask] = rgb_pred
    img_gt = np.zeros((H, W, 3)) + white_bkgd
    img_gt[mask] = rgb_gt
    if eval_whole_img:
        rgb_pred, rgb_gt = img_pred, img_gt
    terms = (rgb_pred - rgb_gt) ** 2
    mse = np.mean(terms)
    psnr = -10 * np.log(mse) / np.log(10)
    mse_f64 = math.fsum(terms.astype(np.float64).ravel()) / terms.size if terms.size else float("nan")
    if eval_whole_img:
        box = (0, 0, W, H)
    elif png_dir is not None:
        import cv2
        box = tuple(int(v) for v in cv2.boundingRect(mask.astype(np.uint8)))
    else:
        box = bounding_rect(mask)
    x, y, w, h = box
    crop_pred, crop_gt = img_pred[y:y + h, x:x + w], img_gt[y:y + h, x:x + w]
    out = {"mse": mse, "psnr": psnr, "mse_f64": mse_f64, "box": box,
           "crop_pred": to_u8(crop_pred[..., [2, 1, 0]] * 255), "crop_gt": to_u8(crop_gt[..., [2, 1, 0]] * 255)}
    if png_dir is not None:
        import cv2
        cv2.imwrite(os.path.join(png_dir, 'frame{:04d}_view{:04d}.png'.format(frame_index, view_index)),
                    crop_pred[..., [2, 1, 0]] * 255)
        cv2.imwrite(os.path.join(png_dir, 'frame{:04d}_view{:04d}_gt.png'.format(frame_index, view_index)),
                    crop_gt[..., [2, 1, 0]] * 255)
    out["ssim"] = compare_ssim(crop_pred, crop_gt, multichannel=True)
    return out
