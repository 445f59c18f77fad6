"""The demo visualizers' frame restated in numpy (TEST INFRASTRUCTURE ONLY): what upstream's lib/visualizers/if_nerf_demo.py
and if_nerf_perform.py hand cv2.imwrite, as the uint8 array cv2 stores.  nb_vis_frame computes the same bytes on the GPU."""
import numpy as np

from oracle.eval_metrics import to_u8


def float_image(rgb_map, mask_at_box, H, W, white_bkgd=False):
    """Upstream's float64 image before imwrite (if_nerf_demo.py:16-26, :52): zeros (+ 1 with white_bkgd), the rays
    scattered into the mask's pixels in row-major order, BGR, times 255.  numpy raises upstream's ValueErrors: the reshape of
    a mask whose size is not H * W, and the "shape mismatch" of a ray count the mask does not take."""
    mask = np.asarray(mask_at_box).reshape(H, W)
    img = np.zeros((H, W, 3))
    if white_bkgd:
        img = img + 1
    img[mask] = np.asarray(rgb_map)
    return img[..., [2, 1, 0]] * 255


def frame(rgb_map, mask_at_box, H, W, white_bkgd=False):
    """The (H,W,3) uint8 BGR array cv2.imwrite stores for float_image."""
    return to_u8(float_image(rgb_map, mask_at_box, H, W, white_bkgd))
