"""f-2: camera rays on the device.  Replaces lib/utils/render_utils.py:120-137 (`image_rays`: get_rays + get_near_far +
mask_at_box compaction), which upstream runs in numpy per view and ships to the GPU (8.4 MB per 512x512 view)."""
import ctypes as C

import numpy as np
import torch

from . import capi


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
    f64, host = _camera_operands(RT, K)
    if bounds.dtype != np.float32 or bounds.shape != (2, 3):
        raise ValueError("bounds must be the float32 (2,3) can_bounds (got %s %s)" % (bounds.dtype, bounds.shape))
    return _image_rays_call(host, f64, False, bounds, H, W, device)


def _camera_operands(RT, K):
    """The host operands of nb_image_rays / nb_image_rays_f64 for the numpy camera RT (3,4) or (4,4), K (3,3), both float32
    or both float64: -> (f64, [K_inv, R, T, o]) in the camera's dtype, inv(K) and the camera centre -np.dot(R.T, T) by
    upstream's own numpy expressions (get_rays :10 and :16)."""
    if RT.dtype != K.dtype or RT.dtype not in (np.float32, np.float64):
        raise ValueError("the camera must be all float32 or all float64 (got RT %s, K %s)" % (RT.dtype, K.dtype))
    if RT.shape not in ((3, 4), (4, 4)) or K.shape != (3, 3):
        raise ValueError("RT must be (3,4) or (4,4) and K (3,3) (got %s and %s)" % (RT.shape, K.shape))
    R, T = RT[:3, :3], RT[:3, 3]
    return RT.dtype == np.float64, [np.ascontiguousarray(x, dtype=RT.dtype).reshape(-1)
                                    for x in (np.linalg.inv(K), R, T, -np.dot(R.T, T).ravel())]


def _image_rays_enqueue(a, host, f64, dev):
    """Enqueue nb_image_rays_f64 (f64) or nb_image_rays with the args `a` and the host operands `host` (K_inv, R, T, o) on
    the current stream of `dev`."""
    lib = capi.load()
    ct = C.c_double if f64 else C.c_float
    fn, name = (lib.nb_image_rays_f64, "nb_image_rays_f64") if f64 else (lib.nb_image_rays, "nb_image_rays")
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        capi.check(fn(C.byref(a), *[x.ctypes.data_as(C.POINTER(ct)) for x in host], stream), name)


class ShardedRays:
    """Fixed-shape device buffers for one rank's interleaved shard of an H x W view (nb_image_rays' shard mode): nothing is
    compacted, so generating the rays of the next view from a camera on the host never synchronises with it.  A box-hit ray
    carries the bits camera_image_rays gives its pixel; rays that miss the box (upstream drops them, render_utils.py:131-132)
    are dead rays with mask 0."""

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
        self._args = a = capi.nb_image_rays_args()
        a.H, a.W, a.rank, a.world, a.chunk, a.n_local = self.H, self.W, self.rank, self.world, self.chunk, self.n_local
        a.ray_o, a.ray_d, a.near, a.far = (t.data_ptr() for t in (self.ray_o, self.ray_d, self.near, self.far))
        a.mask_at_box = self.mask.data_ptr()

    def generate(self, RT, K, bounds):
        """Enqueue the ray generation of one view on the current stream; returns self (ray_o, ray_d, near, far, mask).  RT
        and K as camera_image_rays takes them (a float64 camera runs nb_image_rays_f64, a float32 one nb_image_rays);
        bounds, the world box (2,3), is cast to float32."""
        f64, host = _camera_operands(*_host(RT, K))
        self._args.bounds[:] = np.asarray(bounds, dtype=np.float32).reshape(-1).tolist()
        _image_rays_enqueue(self._args, host, f64, self.ray_o.device)
        return self


def _image_rays_call(host, f64, k_f32, bounds, H, W, device, image=None):
    """One nb_image_rays / nb_image_rays_f64 call on the host operands `host` (K_inv, R, T, o) -> ray_o, ray_d, near, far,
    mask_at_box and, with `image` (a device (H,W,3) float32 tensor), rgb."""
    lib = capi.load()
    H, W = int(H), int(W)
    nbytes = lib.nb_image_rays_workspace_bytes(H, W)
    if nbytes == 0:
        raise ValueError("bad image size %d x %d" % (H, W))
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
        for i, v in enumerate(np.asarray(bounds, dtype=np.float32).reshape(-1)):
            a.bounds[i] = float(v)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        a.ray_o, a.ray_d, a.near, a.far = ray_o.data_ptr(), ray_d.data_ptr(), near.data_ptr(), far.data_ptr()
        a.mask_at_box, a.count = mask.data_ptr(), count.data_ptr()
        rgb = None
        if image is not None:
            if tuple(image.shape) != (H, W, 3) or image.dtype != torch.float32:
                raise ValueError("image must be (H,W,3) float32 (got %s %s)" % (tuple(image.shape), image.dtype))
            image = image.to(dev).contiguous()
            rgb = torch.empty((n, 3), dtype=torch.float32, device=dev)
            a.image, a.rgb = image.data_ptr(), rgb.data_ptr()
        a.k_f32 = 1 if k_f32 else 0
        _image_rays_enqueue(a, host, f64, dev)
        m = int(count.item())
        out = (ray_o[:m], ray_d[:m], near[:m], far[:m], mask.bool())
        return out if rgb is None else out + (rgb[:m],)


def dataset_image_rays(cam, k_kind, H, W, image, device="cuda:0"):
    """if_nerf_data_utils.sample_ray / sample_ray_h36m for split 'test' (:138-148 / :220-230) on the device: get_rays over
    the view, `.astype(np.float32)`, get_near_far in float32 and the mask_at_box compaction of the rays and of the image's
    colours, bit for bit (nb_image_rays_f64; People-Snapshot's float32 K with `k_f32`).  cam: the (NB_TRAIN_CAM_DOUBLES,)
    float64 camera of `train_camera` (upstream's inv(K) and camera centre, its float32 box); image: the (H,W,3) float32
    device tensor.  -> ray_o, ray_d (n,3), near, far (n,), mask_at_box (H*W,) bool, rgb (n,3)."""
    cam = np.asarray(cam, dtype=np.float64).reshape(-1)
    if cam.shape != (capi.NB_TRAIN_CAM_DOUBLES,):
        raise ValueError("cam must be the (%d,) train_camera array" % capi.NB_TRAIN_CAM_DOUBLES)
    host = [np.ascontiguousarray(cam[a:b]) for a, b in ((0, 9), (9, 18), (18, 21), (21, 24))]
    return _image_rays_call(host, True, int(k_kind) == capi.NB_SCALAR_F32, cam[24:30].astype(np.float32), H, W, device,
                            image=image)


def train_camera(K, R, T, can_bounds):
    """The per-item camera nb_train_rays reads, from the operands upstream's sample_ray / sample_ray_h36m receive: K (3,3)
    in its dtype (float32 for People-Snapshot, float64 for ZJU-MoCap), R (3,3) and T (3,1) float64, the float32 can_bounds
    (2,3).  inv(K) and the camera centre -np.dot(R.T, T) are upstream's own expressions on these operands (get_rays :10 and
    :16; the centre's rounding depends on the operands' layout, so call this with the arrays upstream has).  -> (k_kind,
    (NB_TRAIN_CAM_DOUBLES,) float64), every value exact in its kind."""
    K, R, T, can_bounds = (np.asarray(x) for x in (K, R, T, can_bounds))
    if K.shape != (3, 3) or K.dtype not in (np.float32, np.float64):
        raise ValueError("K must be a float32 or float64 (3,3) (got %s %s)" % (K.dtype, K.shape))
    if R.shape != (3, 3) or R.dtype != np.float64 or T.size != 3 or T.dtype != np.float64:
        raise ValueError("R (3,3) and T (3,1) must be float64, as the training datasets hand them to get_rays "
                         "(got %s %s, %s %s)" % (R.dtype, R.shape, T.dtype, T.shape))
    if can_bounds.dtype != np.float32 or can_bounds.shape != (2, 3):
        raise ValueError("can_bounds must be the float32 (2,3) box (got %s %s)" % (can_bounds.dtype, can_bounds.shape))
    o = -np.dot(R.T, T).ravel()
    cam = np.concatenate([np.linalg.inv(K).astype(np.float64).ravel(), R.ravel(), T.ravel(), o,
                          can_bounds.astype(np.float64).ravel()])
    kind = capi.NB_SCALAR_F32 if K.dtype == np.float32 else capi.NB_SCALAR_F64
    return kind, cam


_STATUS = {capi.NB_TRAIN_RAYS_ROUNDS: "no N_rand rays after %d sampling rounds: the bound pixels' rays miss the box (upstream "
                                      "loops forever here)" % capi.NB_TRAIN_RAYS_MAX_ROUNDS,
           capi.NB_TRAIN_RAYS_EMPTY: "a class the round draws from has no pixels (upstream's np.random.randint raises here)",
           capi.NB_TRAIN_RAYS_REPLAY: "the replayed draws do not fit the pixel lists"}


class EmptyClassError(RuntimeError, ValueError):
    """A failed nb_train_rays item whose round drew from an empty class list: where upstream's item raises ValueError
    (np.random.randint), so it is a ValueError as well as the RuntimeError of any failed call."""


class TrainRays:
    """The device outputs of one nb_train_rays call, (B, n_rays, ...) each, and its per-item status.  The status comes to
    pinned host memory with the stream's work; `check()` waits for it (free once something has synchronised the stream past
    the call, as Renderer.render does by checking after prepare_sp_input's `.tolist()`) and raises RuntimeError for a failed
    item."""

    def __init__(self, ray_o, ray_d, near, far, rgb, coord, rounds, status, status_host):
        self.ray_o, self.ray_d, self.near, self.far, self.rgb = ray_o, ray_d, near, far, rgb
        self.coord, self.rounds, self.status = coord, rounds, status
        self._status_host, self._event = status_host, torch.cuda.Event()
        self._event.record(torch.cuda.current_stream(status.device))

    def check(self):
        self._event.synchronize()
        for b, s in enumerate(self._status_host.tolist()):
            if s != capi.NB_TRAIN_RAYS_OK:
                raise (EmptyClassError if s == capi.NB_TRAIN_RAYS_EMPTY else RuntimeError)("nb_train_rays: batch item %d: %s" % (b, _STATUS.get(s, "status %d" % s)))
        return self


def train_rays(image, class_map, cams, k_kind, n_rays, body_ratio, face_ratio, draws=None, want_coord=False):
    """if_nerf_data_utils.sample_ray_h36m / sample_ray, split 'train', on the device (nb_train_rays), for a batch of B items.
    image (B,H,W,3) float32 and class_map (B,H,W) uint8 (NB_TRAIN_CLASS_* bits), CUDA tensors on one device; cams
    (B, NB_TRAIN_CAM_DOUBLES) float64 on the host (stacked `train_camera` results) and their k_kind.  Randomness: `draws`
    None keys the kernel's Philox with two 64-bit words drawn from torch's CPU default generator (so torch.manual_seed makes
    the call reproducible and the CUDA generator is left alone); otherwise a list of B int64 arrays, the np.random.randint
    results upstream drew for each item, rounds concatenated (replay, for tests).  Nothing here synchronises with the host.
    -> TrainRays."""
    lib = capi.load()
    if not (torch.is_tensor(image) and torch.is_tensor(class_map)) or image.device.type != "cuda":
        raise ValueError("image and class_map must be CUDA tensors")
    dev = image.device
    B, H, W = int(class_map.shape[0]), int(class_map.shape[1]), int(class_map.shape[2])
    if tuple(image.shape) != (B, H, W, 3) or image.dtype != torch.float32 or class_map.dtype != torch.uint8 \
            or class_map.device != dev:
        raise ValueError("image must be (B,H,W,3) float32 and class_map (B,H,W) uint8 on one device (got %s %s, %s %s)"
                         % (tuple(image.shape), image.dtype, tuple(class_map.shape), class_map.dtype))
    cams = np.ascontiguousarray(cams, dtype=np.float64)
    if cams.shape != (B, capi.NB_TRAIN_CAM_DOUBLES):
        raise ValueError("cams must be (B, %d) (got %s)" % (capi.NB_TRAIN_CAM_DOUBLES, cams.shape))
    nbytes = lib.nb_train_rays_workspace_bytes(B, H, W)
    if nbytes == 0:
        raise ValueError("bad batch size %d x %d x %d" % (B, H, W))
    n = int(n_rays)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        a = capi.nb_train_rays_args()
        a.B, a.H, a.W, a.n_rays = B, H, W, n
        a.body_ratio, a.face_ratio = float(body_ratio), float(face_ratio)
        a.k_kind, a.rt_kind = int(k_kind), capi.NB_SCALAR_F64
        image, class_map = image.contiguous(), class_map.contiguous()
        a.image, a.class_map = image.data_ptr(), class_map.data_ptr()
        cams_dev = torch.from_numpy(cams).pin_memory().to(dev, non_blocking=True)
        a.cams = cams_dev.data_ptr()
        if draws is None:
            key = torch.randint(-2 ** 63, 2 ** 63 - 1, (2,), dtype=torch.int64).numpy().view(np.uint64)
            a.key[0], a.key[1] = int(key[0]), int(key[1])
        else:
            if len(draws) != B:
                raise ValueError("draws must hold one array per batch item")
            off = np.concatenate([[0], np.cumsum([len(d) for d in draws])]).astype(np.int64)
            flat = np.concatenate([np.asarray(d, dtype=np.int64).ravel() for d in draws] + [np.zeros(1, np.int64)])
            dd = torch.from_numpy(flat).pin_memory().to(dev, non_blocking=True)
            do = torch.from_numpy(off).pin_memory().to(dev, non_blocking=True)
            a.draws, a.draw_offset = dd.data_ptr(), do.data_ptr()
        out = [torch.empty((B, n, 3), dtype=torch.float32, device=dev) for _ in range(2)] + \
              [torch.empty((B, n), dtype=torch.float32, device=dev) for _ in range(2)] + \
              [torch.empty((B, n, 3), dtype=torch.float32, device=dev)]
        a.ray_o, a.ray_d, a.near, a.far, a.rgb = (t.data_ptr() for t in out)
        coord = torch.empty((B, n), dtype=torch.int32, device=dev) if want_coord else None
        a.coord = coord.data_ptr() if coord is not None else None
        rounds = torch.empty((B,), dtype=torch.int32, device=dev)
        status = torch.empty((B,), dtype=torch.int32, device=dev)
        a.rounds, a.status = rounds.data_ptr(), status.data_ptr()
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        capi.check(lib.nb_train_rays(C.byref(a), C.c_void_p(stream.cuda_stream)), "nb_train_rays")
        status_host = torch.empty((B,), dtype=torch.int32, pin_memory=True)
        status_host.copy_(status, non_blocking=True)
        return TrainRays(*out, coord, rounds, status, status_host)
