"""f-2: camera rays on the device.  Replaces lib/utils/render_utils.py:120-137 (`image_rays`: get_rays + get_near_far +
mask_at_box compaction), which upstream runs in numpy per view and ships to the GPU (8.4 MB per 512x512 view)."""
import ctypes as C

import numpy as np
import torch

from . import capi


def _camera(RT, K, bounds, H, W):
    RT = np.asarray(RT, dtype=np.float64)
    cam = capi.nb_camera()
    kinv = np.linalg.inv(np.asarray(K, dtype=np.float64))
    for i, v in enumerate(kinv.reshape(-1)):
        cam.K_inv[i] = float(v)
    for i, v in enumerate(RT[:3, :3].reshape(-1)):
        cam.R[i] = float(v)
    for i, v in enumerate(RT[:3, 3].reshape(-1)):
        cam.T[i] = float(v)
    for i, v in enumerate(np.asarray(bounds, dtype=np.float32).astype(np.float64).reshape(-1)):
        cam.bounds[i] = float(v)
    cam.H, cam.W = int(H), int(W)
    return cam


class ShardedRays:
    """Fixed-shape device buffers for one rank's interleaved shard of an H x W view (nb_gen_rays_sharded): nothing is
    compacted, so generating the rays of the next view never synchronises with the host.  Rays that miss the box (upstream
    drops them, render_utils.py:131-132) are dead rays with mask 0."""

    def __init__(self, H, W, rank=0, world=1, chunk=256, device="cuda:0"):
        self.H, self.W, self.rank, self.world, self.chunk = int(H), int(W), int(rank), int(world), int(chunk)
        n = self.H * self.W
        n_chunks = (n + chunk - 1) // chunk
        self.n_local = ((n_chunks + world - 1) // world) * chunk
        dev = torch.device(device)
        self.ray_o = torch.empty((1, self.n_local, 3), dtype=torch.float32, device=dev)
        self.ray_d = torch.empty((1, self.n_local, 3), dtype=torch.float32, device=dev)
        self.near = torch.empty((1, self.n_local), dtype=torch.float32, device=dev)
        self.far = torch.empty((1, self.n_local), dtype=torch.float32, device=dev)
        self.mask = torch.empty((1, self.n_local), dtype=torch.uint8, device=dev)
        self.lib = capi.load()

    def generate(self, RT, K, bounds):
        """Enqueue the ray generation of one view on the current stream; returns self (ray_o, ray_d, near, far, mask)."""
        cam = _camera(RT, K, bounds, self.H, self.W)
        dev = self.ray_o.device
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(self.lib.nb_gen_rays_sharded(C.byref(cam), self.rank, self.world, self.chunk, self.n_local,
                                                    self.ray_o.data_ptr(), self.ray_d.data_ptr(), self.near.data_ptr(),
                                                    self.far.data_ptr(), self.mask.data_ptr(), C.c_void_p(stream)),
                       "nb_gen_rays_sharded")
        return self


def _host(*xs):
    """numpy copies of numpy arrays / tensors.  The device tensors among them come over in ONE copy (widened to float64,
    which holds float32 values exactly, and narrowed back), so a camera left on the GPU costs one host synchronisation."""
    dev = [x for x in xs if torch.is_tensor(x) and x.device.type != "cpu"]
    flat = torch.cat([x.detach().reshape(-1).to(torch.float64) for x in dev]).cpu().numpy() if dev else None
    out, at = [], 0
    for x in xs:
        if torch.is_tensor(x) and x.device.type != "cpu":
            n = x.numel()
            out.append(flat[at:at + n].reshape(tuple(x.shape)).astype(str(x.dtype).replace("torch.", "")))
            at += n
        else:
            out.append(x.detach().numpy() if torch.is_tensor(x) else np.asarray(x))
    return out


def camera_image_rays(RT, K, bounds, H, W, device="cuda:0"):
    """render_utils.image_rays (render_utils.py:120-137) bit for bit, on the device (nb_image_rays / nb_image_rays_f64).
    RT (3,4) or (4,4) world->camera and K (3,3), both float32 or both float64 as the dataset holds them (numpy arrays or
    tensors); bounds (2,3) the float32 can_bounds; H, W the image size.  -> ray_o, ray_d (n,3), near, far (n,) float32 and
    mask_at_box (H*W,) bool, torch tensors on `device`, in row-major pixel order.  inv(K) and the camera centre
    -np.dot(R.T, T) are computed here with upstream's own numpy expressions, so the camera is needed on the host: a camera
    given on the host costs one host synchronisation (reading n), one given as device tensors two (one copy of all of it
    to the host, then n)."""
    RT, K, bounds = _host(RT, K, bounds)
    if RT.dtype != K.dtype or RT.dtype not in (np.float32, np.float64):
        raise ValueError("the camera must be all float32 or all float64 (got RT %s, K %s)" % (RT.dtype, K.dtype))
    if RT.shape not in ((3, 4), (4, 4)) or K.shape != (3, 3):
        raise ValueError("RT must be (3,4) or (4,4) and K (3,3) (got %s and %s)" % (RT.shape, K.shape))
    if bounds.dtype != np.float32 or bounds.shape != (2, 3):
        raise ValueError("bounds must be the float32 (2,3) can_bounds (got %s %s)" % (bounds.dtype, bounds.shape))
    lib = capi.load()
    H, W = int(H), int(W)
    nbytes = lib.nb_image_rays_workspace_bytes(H, W)
    if nbytes == 0:
        raise ValueError("bad image size %d x %d" % (H, W))
    f64 = RT.dtype == np.float64
    ct = C.c_double if f64 else C.c_float
    R, T = RT[:3, :3], RT[:3, 3]
    host = [np.ascontiguousarray(x, dtype=RT.dtype).reshape(-1)
            for x in (np.linalg.inv(K), R, T, -np.dot(R.T, T).ravel())]   # get_rays :10 and :16, as upstream evaluates them
    ptrs = [x.ctypes.data_as(C.POINTER(ct)) for x in host]
    dev = torch.device(device)
    n = H * W
    with torch.cuda.device(dev):
        ray_o = torch.empty((n, 3), dtype=torch.float32, device=dev)
        ray_d = torch.empty((n, 3), dtype=torch.float32, device=dev)
        near = torch.empty((n,), dtype=torch.float32, device=dev)
        far = torch.empty((n,), dtype=torch.float32, device=dev)
        mask = torch.empty((n,), dtype=torch.uint8, device=dev)
        count = torch.empty((1,), dtype=torch.int32, device=dev)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        a = capi.nb_image_rays_args()
        a.H, a.W = H, W
        for i, v in enumerate(bounds.reshape(-1)):
            a.bounds[i] = float(v)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        a.ray_o, a.ray_d, a.near, a.far = ray_o.data_ptr(), ray_d.data_ptr(), near.data_ptr(), far.data_ptr()
        a.mask_at_box, a.count = mask.data_ptr(), count.data_ptr()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        fn, name = (lib.nb_image_rays_f64, "nb_image_rays_f64") if f64 else (lib.nb_image_rays, "nb_image_rays")
        capi.check(fn(C.byref(a), *ptrs, stream), name)
        m = int(count.item())
        return ray_o[:m], ray_d[:m], near[:m], far[:m], mask.bool()


def image_rays(RT, K, bounds, H, W, device="cuda:0"):
    """RT (3,4) or (4,4) world->camera, K (3,3), bounds (2,3) world box -> ray_o, ray_d (n,3), near, far (n,), mask_at_box
    (H*W,) bool, all torch tensors on `device`; n = mask_at_box.sum() (order = row-major pixel order, as upstream)."""
    lib = capi.load()
    dev = torch.device(device)
    cam = _camera(RT, K, bounds, H, W)
    n = int(H) * int(W)
    with torch.cuda.device(dev):
        ray_o = torch.empty((n, 3), dtype=torch.float32, device=dev)
        ray_d = torch.empty((n, 3), dtype=torch.float32, device=dev)
        near = torch.empty((n,), dtype=torch.float32, device=dev)
        far = torch.empty((n,), dtype=torch.float32, device=dev)
        mask = torch.empty((n,), dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        capi.check(lib.nb_gen_rays(C.byref(cam), ray_o.data_ptr(), ray_d.data_ptr(), near.data_ptr(), far.data_ptr(),
                                   mask.data_ptr(), C.c_void_p(stream)), "nb_gen_rays")
        m = mask.bool()
        return ray_o[m], ray_d[m], near[m], far[m], m
