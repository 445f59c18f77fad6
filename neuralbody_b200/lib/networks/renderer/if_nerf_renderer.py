"""Drop-in for the reference's Neural Body renderer.

Replaces lib/networks/renderer/if_clight_renderer.py (the file every Neural Body config
selects through `renderer_module/renderer_path`; the project brief calls it
if_nerf_renderer.py): same class name, constructor and `render(batch)` contract
(:94-122), same five output keys/shapes/dtypes (:84-92), same config keys read inside
(`N_samples, perturb, raw_noise_std, white_bkgd` :13,16,82; `voxel_size`
latent_xyzc.py:54).  The body of the per-chunk loop -- get_sampling_points ->
get_density_color -> Network.calculate_density_color -> raw2outputs -- is ONE fused
CUDA launch through the C ABI (include/neuralbody_b200.h); no PyTorch op runs inside
the ray loop and there is no CPU/eager fallback.
"""
import ctypes as C

import torch

from neuralbody_b200 import capi
from neuralbody_b200.lib.config import get_active_cfg

_PRECISIONS = {"fp32": capi.NB_PRECISION_FP32, "tc_fp16": capi.NB_PRECISION_TC_FP16,
               "tc_fp16x3": capi.NB_PRECISION_TC_FP16X3}
# the fields of nb_decoder_weights that point at the 17 tensors of Network.decoder_tensors(), in that order
_DECODER_FIELDS = tuple(f[0] for f in capi.nb_decoder_weights._fields_[:17])


def _input_grad_slots(B, n, S):
    """The eight input-gradient slots after the volumes and the decoder tensors, in _FusedRender.apply order (R, Th, ray_o,
    ray_d, near, far, bounds, z_vals): the nb_render_input_grads field each is accumulated through, and its fp32 shape."""
    return (("d_R", (B, 3, 3)), ("d_Th", (B, 3)), ("d_ray_o", (B, n, 3)), ("d_ray_d", (B, n, 3)),
            ("d_near", (B, n)), ("d_far", (B, n)), ("d_bounds", (B, 2, 3)), ("d_z_vals", (B, n, S)))


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f32c(t, device):
    return t.to(device=device, dtype=torch.float32).contiguous()


class _FusedRender(torch.autograd.Function):
    """Autograd boundary of the training path (BASELINE config 3): forward = nb_render_fwd with the exact
    kernel + activation record, backward = nb_render_bwd_inputs.  Differentiable outputs: all five maps, rgb_map,
    disp_map, acc_map, depth_map and weights, as upstream's raw2outputs (nerf_net_utils.py:37-45); an output the loss
    does not read costs nothing (its cotangent stays None and the kernels get NULL).  disp_map follows upstream's NaN
    rule: on a ray with acc_map == 0 its gradient is NaN, which reaches ray_d only (see nb_render_bwd_maps).
    Differentiable inputs: the four dense volumes (so gradients keep flowing into the reference's SparseConvNet / code
    embedding), the 17 decoder tensors, the frame transform sp_input['R'] / ['Th'] (pose refinement), the rays
    ray_o / ray_d (camera refinement), and near / far, sp_input['bounds'] and a caller-supplied z_vals (None in the
    slots a call does not have: near / far are not read when z_vals is given)."""

    @staticmethod
    def forward(ctx, renderer, call, *tensors):
        out = renderer._launch(call, save=True)
        ctx.renderer, ctx.call = renderer, call
        ctx.n_vol = len(call["feature_volume"])
        ctx.save_for_backward(*tensors)
        ctx.set_materialize_grads(False)    # no zero (B,n,S) cotangent for a loss that does not read weights
        return out["rgb_map"], out["disp_map"], out["acc_map"], out["depth_map"], out["weights"]

    @staticmethod
    def backward(ctx, d_rgb, d_disp, d_acc, d_depth, d_weights):
        grads = ctx.renderer._launch_bwd(ctx.call, d_rgb, d_depth, d_acc, ctx.needs_input_grad[2:], d_disp=d_disp,
                                         d_weights=d_weights)
        return (None, None) + tuple(grads)


class Renderer:
    def __init__(self, net):
        self.net = net
        self.lib = capi.load()
        self._vol_key = None
        self._vol_blob = None
        self._vol_dims = None
        self._vol_dtype = None
        self._w_key = None
        self._w_blob = None
        self._vol_keep = None
        self._w_keep = None
        self._tvals = {}
        self.launches = 0          # render kernels enqueued so far (bench accounting)

    # ------------------------------------------------------------------ options
    def _opt(self, name, default):
        cfg = get_active_cfg()
        return cfg[name] if name in cfg else default

    def _precision(self, key, default):
        """NB_PRECISION_* named by cfg[key] (render_precision, density_precision)."""
        name = str(self._opt(key, default))
        if name not in _PRECISIONS:
            raise ValueError("cfg.%s must be one of %s" % (key, sorted(_PRECISIONS)))
        return _PRECISIONS[name]

    def _train_precision(self, B, n, S):
        """Precision of a call autograd records: 'tc_tf32x3' (default: sample list + wgmma TF32 GEMM chains, exact empty-sample
        skipping in forward and backward) or 'fp32' (the exact FFMA kernels)."""
        name = str(self._opt("render_train_precision", "tc_tf32x3"))
        if name not in ("tc_tf32x3", "fp32"):
            raise ValueError("cfg.render_train_precision must be 'tc_tf32x3' or 'fp32'")
        if name == "tc_tf32x3" and S <= 256 and B * n * S < (1 << 28) and self.lib.nb_has_precision(capi.NB_PRECISION_TC_TF32X3):
            return capi.NB_PRECISION_TC_TF32X3
        return capi.NB_PRECISION_FP32

    def _volume_dtype(self, precision):
        name = str(self._opt("render_volume_dtype", "auto"))
        if name == "auto":
            # the fp16 volume alone costs ~1e-3 of depth_map parity: only the 1-pass mode gathers from it
            return capi.NB_DTYPE_F16 if precision == capi.NB_PRECISION_TC_FP16 else capi.NB_DTYPE_F32
        return {"fp32": capi.NB_DTYPE_F32, "fp16": capi.NB_DTYPE_F16}[name]

    # ------------------------------------------------------------------ a2 (host API parity)
    def get_sampling_points(self, ray_o, ray_d, near, far, t_rand=None):
        """if_clight_renderer.py:11-27, kept callable for subclasses.  `render` does not call
        this: the fused kernel generates the same samples in registers."""
        cfg = get_active_cfg()
        t_vals = torch.linspace(0., 1., steps=cfg.N_samples).to(near)
        z_vals = near[..., None] * (1. - t_vals) + far[..., None] * t_vals
        if cfg.perturb > 0. and self.net.training:
            mids = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
            upper = torch.cat([mids, z_vals[..., -1:]], -1)
            lower = torch.cat([z_vals[..., :1], mids], -1)
            if t_rand is None:
                t_rand = torch.rand(z_vals.shape)
            z_vals = lower + (upper - lower) * t_rand.to(upper)
        pts = ray_o[:, :, None] + ray_d[:, :, None] * z_vals[..., None]
        return pts, z_vals

    # ------------------------------------------------------------------ a3
    def prepare_sp_input(self, batch):
        """if_clight_renderer.py:29-52, unchanged semantics (stays Python; `.tolist()` is the
        one host sync per frame, exactly as upstream)."""
        sp_input = {}
        sh = batch['coord'].shape
        idx = [torch.full([sh[1]], i) for i in range(sh[0])]
        idx = torch.cat(idx).to(batch['coord'])
        coord = batch['coord'].view(-1, sh[-1])
        sp_input['coord'] = torch.cat([idx[:, None], coord], dim=1)
        out_sh, _ = torch.max(batch['out_sh'], dim=0)
        sp_input['out_sh'] = out_sh.tolist()
        sp_input['batch_size'] = sh[0]
        sp_input['bounds'] = batch['bounds']
        sp_input['R'] = batch['R']
        sp_input['Th'] = batch['Th']
        sp_input['latent_index'] = batch['latent_index']
        return sp_input

    def get_density_color(self, wpts, viewdir, raw_decoder):
        """if_clight_renderer.py:54-60 (host API parity for subclasses that pass their own decoder)."""
        n_batch, n_pixel, n_sample = wpts.shape[:3]
        wpts = wpts.view(n_batch, n_pixel * n_sample, -1)
        viewdir = viewdir[:, :, None].repeat(1, 1, n_sample, 1).contiguous()
        viewdir = viewdir.view(n_batch, n_pixel * n_sample, -1)
        return raw_decoder(wpts, viewdir)

    # ------------------------------------------------------------------ once-per-frame packs
    def pack_volume(self, feature_volume, dtype):
        """NCDHW fp32 volumes -> channels-last blob (nb_pack_volume); cached until the tensors change."""
        # the key holds STRONG references to the keyed tensors (self._vol_keep): while an entry is cached, the caching
        # allocator cannot hand the same address to another frame's volumes, so (data_ptr, shape, _version) identifies them
        key = (dtype,) + tuple((v.data_ptr(), tuple(v.shape), v._version) for v in feature_volume)
        if key == self._vol_key:
            return self._vol_blob, self._vol_dims
        if len(feature_volume) != capi.NB_NUM_LEVELS:
            raise ValueError("expected %d feature volumes" % capi.NB_NUM_LEVELS)
        dev = feature_volume[0].device
        if dev.type != "cuda":
            raise RuntimeError("feature volumes must live on a CUDA device (no CPU render path)")
        B = feature_volume[0].shape[0]
        dims = capi.LevelDims()
        levels = (capi.nb_volume_level * capi.NB_NUM_LEVELS)()
        keep = []
        for l, v in enumerate(feature_volume):
            v = v.detach()
            if v.dtype != torch.float32 or not v.is_contiguous():
                v = v.float().contiguous()
            keep.append(v)
            _, c, d, h, w = v.shape
            dims[l][0], dims[l][1], dims[l][2], dims[l][3] = c, d, h, w
            levels[l].data = v.data_ptr()
            levels[l].C, levels[l].D, levels[l].H, levels[l].W = c, d, h, w
        nbytes = self.lib.nb_packed_volume_bytes(dims, B, dtype)
        blob = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        capi.check(self.lib.nb_pack_volume(levels, B, dtype, blob.data_ptr(), nbytes, C.c_void_p(stream)),
                   "nb_pack_volume")
        self._vol_key, self._vol_blob, self._vol_dims, self._vol_dtype = key, blob, dims, dtype
        self._vol_keep = list(feature_volume)
        return blob, dims

    def pack_weights(self, latent_index, device):
        """Fold + re-lay-out the decoder (nb_pack_weights); cached on parameter versions.  nb_pack_weights folds the VALUE
        of latent_index into the blob, so the cache keeps a strong reference to the keyed index tensor (self._w_keep): a
        new frame's freshly allocated index can then never alias the cached one's address."""
        tensors = self.net.decoder_tensors()
        key = tuple((t.data_ptr(), t._version) for t in tensors) + (latent_index.data_ptr(), latent_index._version,
                                                                    tuple(latent_index.shape), str(latent_index.device))
        if key == self._w_key:
            return self._w_blob
        B = int(latent_index.shape[0])
        w, keep = self._weights_struct(tensors, latent_index, device)
        nbytes = self.lib.nb_packed_weights_bytes(B)
        blob = torch.empty(nbytes, dtype=torch.uint8, device=device)
        stream = torch.cuda.current_stream(device).cuda_stream
        capi.check(self.lib.nb_pack_weights(C.byref(w), blob.data_ptr(), nbytes, C.c_void_p(stream)), "nb_pack_weights")
        self._w_key, self._w_blob = key, blob
        self._w_keep = (list(tensors), latent_index)
        return blob

    def _t_vals(self, S, device):
        k = (S, str(device))
        if k not in self._tvals:
            # upstream: torch.linspace(0., 1., steps=cfg.N_samples).to(near)  -- computed on the CPU, then moved
            self._tvals[k] = torch.linspace(0., 1., steps=S).to(device)
        return self._tvals[k]

    def _draw_t_rand(self, B, n, S, device):
        """The jitter draw of if_clight_renderer.py:22 (`torch.rand(z_vals.shape).to(upper)`, CPU
        generator), issued per 2048-ray chunk like upstream so the RNG stream is identical."""
        parts = [torch.rand((B, min(2048, n - i), S)) for i in range(0, n, 2048)]
        # (a training chunk is ONE part: no CPU torch.cat, whose OpenMP region is a thread hand-off per step -- on a busy
        # host such wake-ups were measured at 30-60 ms, ten times the GPU time of the step)
        host = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
        return host.to(device).contiguous()

    # ------------------------------------------------------------------ fused launch
    def render_rays(self, ray_o, ray_d, near, far, feature_volume, sp_input, t_rand=None, want_raw=False,
                    out=None, trace=None, masks=None, z_vals=None, want_weights=None):
        """One nb_render_fwd launch for (B,n) rays.  Returns the dict of get_pixel_value.
        When autograd is recording and any volume / decoder tensor, sp_input['R'] / ['Th'] / ['bounds'], ray_o / ray_d,
        near / far (or z_vals, when given) requires grad, the call goes through the training precision and `_FusedRender` so
        that `loss.backward()` works as it does upstream."""
        cfg = get_active_cfg()
        if int(self._opt("xyz_res", 10)) != 10 or int(self._opt("view_res", 4)) != 4:
            # embedder.py:53-54: the kernels (and view_fc's 346 input columns) are built for PE widths 63 / 27
            raise NotImplementedError("cfg.xyz_res / cfg.view_res other than 10 / 4 are not supported by the fused kernels")
        if float(cfg.raw_noise_std) > 0.:
            # upstream's branch draws CPU randn and would crash on GPU tensors (nerf_net_utils.py:33)
            raise NotImplementedError("raw_noise_std > 0 is not supported (it is 0 in every reference config)")
        dev = ray_o.device
        if dev.type != "cuda":
            raise RuntimeError("Renderer.render needs CUDA tensors: the render path has no CPU implementation")
        B, n = int(ray_o.shape[0]), int(ray_o.shape[1])
        S = int(cfg.N_samples) if z_vals is None else int(z_vals.shape[-1])   # z_vals: caller-supplied depths (fine pass, f-4)
        params = self.net.decoder_tensors()
        # the inputs of _input_grad_slots (near / far are not read when the caller gives the depths)
        inputs = [sp_input['R'], sp_input['Th'], ray_o, ray_d, near if z_vals is None else None,
                  far if z_vals is None else None, sp_input['bounds'], z_vals]
        inputs = [t if torch.is_tensor(t) else None for t in inputs]
        needs_grad = torch.is_grad_enabled() and (any(t.requires_grad for t in params) or
                                                  any(v.requires_grad for v in feature_volume) or
                                                  any(t is not None and t.requires_grad for t in inputs))
        precision = self._train_precision(B, n, S) if needs_grad else self._precision("render_precision", "tc_fp16x3")
        skip_empty = bool(self._opt("render_skip_empty", True))
        if precision != capi.NB_PRECISION_FP32 and (S > 1024 or n * S >= (1 << 28)):
            # the tensor-core pipeline works on a frame-wide sample list: rays of up to 1024 samples, < 2^28 samples per frame
            # (every reference config: 64 / 128 samples, <= 1024^2 rays); anything else runs on the exact kernel
            precision = capi.NB_PRECISION_FP32
        if z_vals is not None:
            t_rand = None
        elif t_rand is None and float(cfg.perturb) > 0. and self.net.training:
            t_rand = self._draw_t_rand(B, n, S, dev)
        # the exact kernel's backward reads the fp32 volume only: a call that records activations for it packs that one
        vdtype = capi.NB_DTYPE_F32 if needs_grad and precision == capi.NB_PRECISION_FP32 else self._volume_dtype(precision)
        call = {
            "B": B, "n": n, "S": S, "dev": dev, "precision": precision, "vdtype": vdtype,
            "ray_o": _f32c(ray_o.detach(), dev), "ray_d": _f32c(ray_d.detach(), dev),
            "near": _f32c(near.detach(), dev), "far": _f32c(far.detach(), dev),
            "input_like": [None if t is None else (t.shape, t.dtype, t.device) for t in inputs],
            "sp_input": sp_input, "t_rand": None if t_rand is None else _f32c(t_rand, dev), "white_bkgd": bool(cfg.white_bkgd),
            "z_vals": None if z_vals is None else _f32c(z_vals.detach(), dev),
            "feature_volume": list(feature_volume), "want_raw": want_raw or needs_grad, "user_raw": bool(want_raw), "out": out, "trace": trace,
            "want_weights": (bool(self._opt("render_return_weights", True)) if want_weights is None else bool(want_weights))
                            or needs_grad,
            "skip_empty": skip_empty, "stats": getattr(self, "stats", None),
            "masks": None,
        }
        if masks is not None:   # f-1: mask views of if_clight_renderer_mmsk.py (B = 1 only, as upstream)
            if needs_grad:
                raise NotImplementedError("mask views are an inference feature upstream (vis_novel_view / vis_novel_pose)")
            msks = masks["msks"][0].to(device=dev, dtype=torch.uint8).contiguous()
            snap = None
            if masks.get("R0_snap") is not None:   # single-view variant (if_clight_renderer_msk.py): SMPL -> snapshot world
                snap = (_f32c(masks["R0_snap"][0], dev), _f32c(masks["Th0_snap"][0], dev).reshape(3))
            call["masks"] = (msks, _f32c(masks["RT"][0][:, :3, :4], dev), _f32c(masks["Ks"][0], dev), snap)
        if call["t_rand"] is not None:
            assert tuple(call["t_rand"].shape) == (B, n, S)
        if needs_grad:
            rgb, disp, acc, depth, weights = _FusedRender.apply(self, call, *feature_volume, *params, *inputs)
            ret = {'rgb_map': rgb, 'disp_map': disp, 'acc_map': acc, 'weights': weights, 'depth_map': depth}
            if want_raw:
                ret['raw'] = call["raw"]
            return ret
        return self._launch(call, save=False)

    def _pool_take(self, tag, numel, dtype, dev):
        """A buffer of >= numel elements from the renderer's pool (several can be out at once: the coarse and the fine pass of
        a hierarchical step each hold an activation record until their backward ran)."""
        free = self.__dict__.setdefault("_pool", {}).setdefault((tag, dtype, str(dev)), [])
        fits = [i for i, t in enumerate(free) if t.numel() >= numel]
        if fits:                      # best fit: the coarse pass must not grab the fine pass's (3x larger) record
            return free.pop(min(fits, key=lambda i: free[i].numel()))
        if len(free) >= 4:            # nothing fits and the pool is full: let the allocator have the smallest one back
            free.pop(min(range(len(free)), key=lambda i: free[i].numel()))
        return torch.empty(int(numel), dtype=dtype, device=dev)

    def _pool_give(self, tag, t):
        if t is not None:
            self.__dict__.setdefault("_pool", {}).setdefault((tag, t.dtype, str(t.device)), []).append(t)

    @staticmethod
    def _out_stride(out, B, n):
        """0 for dense output maps; the common ray stride (floats) when the caller's `out` tensors are columns of one fused
        (B,n,stride) record, e.g. the [rgb | disp | acc | depth] slab of neuralbody_b200.dist (nb_render_args.out_ray_stride)."""
        rgb = out['rgb_map']
        if rgb.is_contiguous() and all(out[k].is_contiguous() for k in ('disp_map', 'acc_map', 'depth_map')):
            return 0
        st = int(rgb.stride(1))
        ok = tuple(rgb.shape) == (B, n, 3) and rgb.stride(2) == 1 and rgb.stride(0) == st * n and all(
            tuple(out[k].shape) == (B, n) and out[k].stride(1) == st and out[k].stride(0) == st * n
            for k in ('disp_map', 'acc_map', 'depth_map'))
        if not ok:
            raise ValueError("`out` maps must be dense, or columns of one (B, n, stride) float32 record")
        return st

    def train_listed_samples(self):
        """[(listed, total)] of the most recent training-precision forward calls (the coarse and the fine pass of a hierarchical
        step): how many samples the exact empty-sample skipping left for the GEMM chains.  Synchronises; diagnostics / bench."""
        return [(int(sv[:4].view(torch.int32)[3].item()), total) for sv, total in self.__dict__.get("_train_records", [])]

    def release(self):
        """Drop every pooled / cached device buffer (activation records, backward scratch, workspace, packed blobs).  The pools
        assume ONE stream drives this Renderer (INTEGRATION.md): call this only when no launch of it is in flight."""
        self.__dict__.pop("_pool", None)
        self.__dict__.pop("_ws_cache", None)
        self.__dict__.pop("_train_records", None)
        self._vol_key = self._vol_blob = self._vol_dims = self._vol_keep = None
        self._w_key = self._w_blob = self._w_keep = None

    def _workspace(self, nbytes, dev):
        """Scratch for nb_render_fwd, grown on demand and reused by every later call on this device's stream."""
        cache = self.__dict__.setdefault("_ws_cache", {})
        ws = cache.get(dev)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(int(nbytes), dtype=torch.uint8, device=dev)
            cache[dev] = ws
        return ws

    def _launch(self, call, save):
        """Pack (cached) + one nb_render_fwd on the current stream."""
        dev, B, n, S = call["dev"], call["B"], call["n"], call["S"]
        precision, vdtype = call["precision"], call["vdtype"]
        with torch.cuda.device(dev), torch.no_grad():
            a, frame = self._frame_args(B, call["feature_volume"], call["sp_input"], vdtype, dev)
            t_vals = self._t_vals(S, dev)
            out = call["out"]
            if out is None:
                out = {
                    'rgb_map': torch.empty((B, n, 3), dtype=torch.float32, device=dev),
                    'disp_map': torch.empty((B, n), dtype=torch.float32, device=dev),
                    'acc_map': torch.empty((B, n), dtype=torch.float32, device=dev),
                    'depth_map': torch.empty((B, n), dtype=torch.float32, device=dev),
                }
                if call["want_weights"]:
                    out['weights'] = torch.empty((B, n, S), dtype=torch.float32, device=dev)
            raw = None
            if call["want_raw"]:
                if save and not call.get("user_raw"):
                    # internal to the autograd node: recycled like the activation record (a fresh 1-3 MB tensor per call comes
                    # out of the caching allocator's large pool, where it splits the blocks the 100 MB volume gradients reuse)
                    raw = self._pool_take("raw", B * n * S * 4, torch.float32, dev)[:B * n * S * 4].view(B, n, S, 4)
                else:
                    raw = torch.empty((B, n, S, 4), dtype=torch.float32, device=dev)
            a.n_rays, a.n_samples = n, S
            a.precision = precision
            sv = None
            if save:
                # the activation record (5.2 KB per sample) and the backward scratch are hundreds of MB per training chunk:
                # they are recycled through a small per-renderer pool instead of going back to the allocator every step
                sv = self._pool_take("save", self.lib.nb_render_save_bytes_for(C.byref(a)) // 4, torch.float32, dev)
            a.ray_o, a.ray_d = call["ray_o"].data_ptr(), call["ray_d"].data_ptr()
            a.near, a.far = call["near"].data_ptr(), call["far"].data_ptr()
            a.t_vals = t_vals.data_ptr()
            a.t_rand = call["t_rand"].data_ptr() if call["t_rand"] is not None else None
            a.z_vals = call["z_vals"].data_ptr() if call["z_vals"] is not None else None
            a.white_bkgd = 1 if call["white_bkgd"] else 0
            a.rgb_map, a.disp_map = out['rgb_map'].data_ptr(), out['disp_map'].data_ptr()
            a.acc_map, a.depth_map = out['acc_map'].data_ptr(), out['depth_map'].data_ptr()
            a.out_ray_stride = self._out_stride(out, B, n)
            a.weights = out['weights'].data_ptr() if 'weights' in out else None
            a.raw = raw.data_ptr() if raw is not None else None
            a.save = sv.data_ptr() if sv is not None else None
            a.skip_empty = 1 if call["skip_empty"] else 0
            if call["masks"] is not None:
                msks, RT, Ks, snap = call["masks"]
                a.mask_msks, a.mask_RT, a.mask_Ks = msks.data_ptr(), RT.data_ptr(), Ks.data_ptr()
                if snap is not None:
                    a.mask_R0, a.mask_Th0 = snap[0].data_ptr(), snap[1].data_ptr()
                a.mask_nv, a.mask_H, a.mask_W = int(msks.shape[0]), int(msks.shape[1]), int(msks.shape[2])
            a.stats = call["stats"].data_ptr() if call["stats"] is not None else None
            ws = None
            if precision in (capi.NB_PRECISION_TC_FP16, capi.NB_PRECISION_TC_FP16X3):   # classify -> decoder over the frame's sample list -> composite
                ws = self._workspace(self.lib.nb_render_fwd_workspace_bytes(B, n, S), dev)
                a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
            a.trace = call["trace"].data_ptr() if call["trace"] is not None else None   # diagnostics (tools/trace_timeline.py)
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(self.lib.nb_render_fwd(C.byref(a), C.c_void_p(stream)), "nb_render_fwd")
            self.launches += B * self.lib.nb_render_fwd_launches(precision)
            if save:   # everything nb_render_bwd needs stays alive with the autograd node
                call["args"], call["save"], call["raw"] = a, sv, raw
                if precision == capi.NB_PRECISION_TC_TF32X3:     # diagnostics: list lengths of the last records (train_listed_samples)
                    recs = self.__dict__.setdefault("_train_records", [])
                    recs.append((sv, B * n * S))
                    del recs[:-4]
                # NOT the output tensors: they carry grad_fn -> this call's autograd node -> ctx.call, a reference cycle only the
                # cyclic garbage collector can free (measured: ~7 MB leaked per training step and a 50-130 ms gc pause every few steps)
                call["keep"] = frame + (t_vals,)
        if raw is not None and call["want_raw"] and not save:
            out = dict(out)
            out['raw'] = raw
        return out

    def _launch_bwd(self, call, d_rgb, d_depth, d_acc, needs, d_disp=None, d_weights=None):
        """nb_render_bwd_inputs: gradients for (volumes..., decoder tensors..., R, Th, ray_o, ray_d, near, far, bounds,
        z_vals) in the order of _FusedRender.apply, from the cotangents of the five maps (None: the loss does not read that
        map)."""
        dev, B, n, S = call["dev"], call["B"], call["n"], call["S"]
        if call.get("save") is None:
            raise RuntimeError("the activation record of this render call was already consumed by a backward pass "
                               "(backward twice through the same nb_render_fwd is not supported)")
        params = self.net.decoder_tensors()
        vols = call["feature_volume"]
        with torch.cuda.device(dev), torch.no_grad():
            def cf(t):
                return None if t is None else t.to(device=dev, dtype=torch.float32).contiguous()
            d_rgb, d_depth, d_acc, d_disp, d_weights = cf(d_rgb), cf(d_depth), cf(d_acc), cf(d_disp), cf(d_weights)
            w = self._weights_struct(params, call["sp_input"]['latent_index'], dev)
            # 17 small tensors (they stay in the allocator's small pool), zeroed by one multi-tensor launch
            gparams = [torch.empty_like(t, dtype=torch.float32, device=dev) for t in params]
            torch._foreach_zero_(gparams)
            g = capi.nb_decoder_weights()
            for name, t in zip(_DECODER_FIELDS, gparams):
                setattr(g, name, t.data_ptr())
            g.latent_index, g.num_train_frame, g.batch = w[0].latent_index, w[0].num_train_frame, B
            want_vol = any(needs[:len(vols)])
            gvols = [torch.zeros_like(v, dtype=torch.float32, device=dev) for v in vols] if want_vol else [None] * len(vols)
            nbytes = self.lib.nb_render_bwd_workspace_bytes_for(C.pointer(call["args"]))
            ws = self._pool_take("bwd_ws", nbytes, torch.uint8, dev)
            ba = capi.nb_render_bwd_args()
            ba.fwd = C.pointer(call["args"])
            ba.save, ba.raw = call["save"].data_ptr(), call["raw"].data_ptr()
            ba.d_rgb_map = d_rgb.data_ptr() if d_rgb is not None else None
            ba.d_depth_map = d_depth.data_ptr() if d_depth is not None else None
            ba.d_acc_map = d_acc.data_ptr() if d_acc is not None else None
            ba.weights, ba.grads = C.pointer(w[0]), C.pointer(g)
            for l in range(capi.NB_NUM_LEVELS):
                ba.d_volumes[l] = gvols[l].data_ptr() if want_vol else None
            ba.workspace, ba.workspace_bytes = ws.data_ptr(), nbytes
            # fp32 accumulators, only for the inputs autograd asks about (pose and camera refinement, depths, box)
            k0 = len(vols) + len(params)
            ig = capi.nb_render_input_grads()
            dins = []
            for (name, shape), want in zip(_input_grad_slots(B, n, S), needs[k0:]):
                d = torch.zeros(shape, dtype=torch.float32, device=dev) if want else None
                setattr(ig, name, d.data_ptr() if d is not None else None)
                dins.append(d)
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(self.lib.nb_render_bwd_inputs(C.byref(ba), _ptr(d_disp), _ptr(d_weights), C.byref(ig),
                                                     C.c_void_p(stream)), "nb_render_bwd_inputs")
            # stream-ordered reuse: the next forward / backward on this stream runs after the kernels just enqueued
            self._pool_give("bwd_ws", ws)
            self._pool_give("save", call.pop("save"))
            if not call.get("user_raw"):
                r = call.pop("raw")
                self._pool_give("raw", r._base if r._base is not None else r)
        # the caller's shape, dtype and device (Th: (B,1,3) or (B,3))
        dins = [None if d is None else d.to(device=like[2], dtype=like[1]).view(like[0])
                for d, like in zip(dins, call["input_like"])]
        grads = list(gvols) + [gp.view_as(t) for gp, t in zip(gparams, params)] + dins
        return [gr if need else None for gr, need in zip(grads, needs)]

    def _weights_struct(self, tensors, latent_index, device):
        """nb_decoder_weights over the raw parameter tensors (+ the tensors kept alive)."""
        w = capi.nb_decoder_weights()
        keep = []
        for name, t in zip(_DECODER_FIELDS, tensors):
            t = t.detach()
            if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
                t = t.to(device=device, dtype=torch.float32).contiguous()
            keep.append(t)
            setattr(w, name, t.data_ptr())
        li = latent_index.to(device=device, dtype=torch.int64).contiguous()
        keep.append(li)
        w.latent_index = li.data_ptr()
        w.num_train_frame = int(self.net.latent.weight.shape[0])
        w.batch = int(latent_index.shape[0])
        return w, keep

    def _frame_args(self, B, feature_volume, sp_input, vdtype, dev):
        """nb_render_args with the frame fields every entry point reads filled in: batch, R, Th, bounds, voxel_size, out_sh
        and the packed volume (level_dims, volume_blob / dtype) and weights.  Returns (args, tensors the args point into):
        the caller keeps those alive while any call reads the args (nb_render_bwd reads R / Th / bounds again)."""
        cfg = get_active_cfg()
        vol_blob, dims = self.pack_volume(feature_volume, vdtype)
        w_blob = self.pack_weights(sp_input['latent_index'], dev)
        R, Th = _f32c(sp_input['R'], dev), _f32c(sp_input['Th'], dev).reshape(B, 3)   # Th: (B,1,3) or (B,3) upstream
        bounds = _f32c(sp_input['bounds'], dev)
        a = capi.nb_render_args()
        a.batch = B
        a.R, a.Th, a.bounds = R.data_ptr(), Th.data_ptr(), bounds.data_ptr()
        for i in range(3):
            a.voxel_size[i] = float(cfg.voxel_size[i])
            a.out_sh[i] = int(sp_input['out_sh'][i])
        for l in range(capi.NB_NUM_LEVELS):
            for j in range(4):
                a.level_dims[l][j] = dims[l][j]
        a.volume_blob, a.volume_dtype, a.weights_blob = vol_blob.data_ptr(), vdtype, w_blob.data_ptr()
        return a, (vol_blob, w_blob, R, Th, bounds)

    def calculate_density(self, wpts, feature_volume, sp_input):
        """Network.calculate_density (latent_xyzc.py:74-89) on arbitrary world points: (B,P,3) -> (B,P,1), raw sigma.
        f-3: the alpha decoder of the mesh renderer (if_mesh_renderer.py:36-41).  `cfg.density_precision`: 'fp32' (default,
        the exact kernel nb_decode_density), or 'tc_fp16x3' / 'tc_fp16' (nb_decode_density_list on the tensor cores; with
        `cfg.render_skip_empty` a point with all-zero features gets sigma(empty) without running the decoder)."""
        dev = wpts.device
        if dev.type != "cuda":
            raise RuntimeError("calculate_density needs CUDA tensors: there is no CPU implementation")
        precision = self._precision("density_precision", "fp32")
        vdtype = capi.NB_DTYPE_F32 if precision == capi.NB_PRECISION_FP32 else self._volume_dtype(precision)
        B, Pn = int(wpts.shape[0]), int(wpts.shape[1])
        with torch.cuda.device(dev), torch.no_grad():
            a, keep = self._frame_args(B, feature_volume, sp_input, vdtype, dev)
            pts = _f32c(wpts, dev)
            sigma = torch.empty((B, Pn, 1), dtype=torch.float32, device=dev)
            a.precision = precision
            stream = torch.cuda.current_stream(dev).cuda_stream
            if precision == capi.NB_PRECISION_FP32:
                capi.check(self.lib.nb_decode_density(C.byref(a), pts.data_ptr(), Pn, sigma.data_ptr(), C.c_void_p(stream)),
                           "nb_decode_density")
                self.launches += 1
            else:   # per frame: classify the points -> decoder over the listed ones
                stats = getattr(self, "stats", None)
                a.skip_empty = 1 if bool(self._opt("render_skip_empty", True)) else 0
                a.stats = stats.data_ptr() if stats is not None else None
                ws = self._workspace(self.lib.nb_decode_density_workspace_bytes(B, Pn), dev)
                a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
                capi.check(self.lib.nb_decode_density_list(C.byref(a), pts.data_ptr(), Pn, sigma.data_ptr(),
                                                           C.c_void_p(stream)), "nb_decode_density_list")
                self.launches += B * (2 + (stats is not None))
        return sigma

    def get_pixel_value(self, ray_o, ray_d, near, far, feature_volume, sp_input, batch):
        """if_clight_renderer.py:62-92: same signature, same returned dict.  With `cfg.render_importance > 0` the call runs the
        coarse + fine passes of `render_rays_hierarchical` and the dict also carries rgb0 / disp0 / acc0 / z_std."""
        if int(self._opt("render_importance", 0)) > 0:
            return self.render_rays_hierarchical(ray_o, ray_d, near, far, feature_volume, sp_input)
        return self.render_rays(ray_o, ray_d, near, far, feature_volume, sp_input)

    # ------------------------------------------------------------------ f-4: hierarchical (coarse + importance) sampling
    def importance_z_vals(self, near, far, weights, n_samples, n_importance, t_rand=None, u=None):
        """z_vals_mid + sample_pdf + sort-merge (volume_renderer.py:84-93, nerf_net_utils.py:55-90) as one nb_sample_pdf launch.
        weights (B,n,S) from the coarse pass; t_rand its jitter (or None); u (B,n,n_importance) uniforms or None for the
        deterministic branch.  Returns (z_all (B,n,S+n_importance) ascending, z_samples (B,n,n_importance)).
        When autograd is recording and near or far requires grad, z_all is an autograd node: as upstream's
        sort(cat(z_vals, z_samples.detach())), each entry that came from the coarse depths (nb_sample_pdf_src says which)
        passes its gradient to that coarse depth and so to near / far; the importance samples get none."""
        dev = weights.device
        B, n, S = int(weights.shape[0]), int(weights.shape[1]), int(n_samples)
        Ni = int(n_importance)
        routed = torch.is_grad_enabled() and (near.requires_grad or far.requires_grad)
        with torch.cuda.device(dev), torch.no_grad():
            z_all = torch.empty((B, n, S + Ni), dtype=torch.float32, device=dev)
            z_smp = torch.empty((B, n, Ni), dtype=torch.float32, device=dev)
            z_src = torch.empty((B, n, S + Ni), dtype=torch.int32, device=dev) if routed else None
            keep = [_f32c(near.detach(), dev), _f32c(far.detach(), dev), self._t_vals(S, dev), _f32c(weights.detach(), dev),
                    None if t_rand is None else _f32c(t_rand, dev), None if u is None else _f32c(u, dev)]
            a = capi.nb_importance_args()
            a.n_rays_total, a.n_samples, a.n_importance = B * n, S, Ni
            a.near, a.far, a.t_vals, a.weights = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr()
            a.t_rand = keep[4].data_ptr() if keep[4] is not None else None
            a.u = keep[5].data_ptr() if keep[5] is not None else None
            a.z_out, a.z_samples = z_all.data_ptr(), z_smp.data_ptr()
            stream = torch.cuda.current_stream(dev).cuda_stream
            if routed:
                capi.check(self.lib.nb_sample_pdf_src(C.byref(a), z_src.data_ptr(), C.c_void_p(stream)), "nb_sample_pdf_src")
            else:
                capi.check(self.lib.nb_sample_pdf(C.byref(a), C.c_void_p(stream)), "nb_sample_pdf")
            self.launches += 1
        if routed:
            # z_all + (c - c.detach()): the value stays the kernel's bit for bit, the gradient reaches the coarse depths
            src = z_src.long()
            zc = self._coarse_z(near, far, S, t_rand, dev).gather(-1, src.clamp(min=0))
            zc = torch.where(src >= 0, zc, torch.zeros_like(zc))
            z_all = z_all + (zc - zc.detach())
        return z_all, z_smp

    def _coarse_z(self, near, far, S, t_rand, dev):
        """The coarse pass's depths as differentiable torch ops of near / far (if_clight_renderer.py:13-23; the kernels derive
        the same values in z_sample): (B,n,S)."""
        near, far = near.to(device=dev, dtype=torch.float32), far.to(device=dev, dtype=torch.float32)
        t_vals = self._t_vals(S, dev)
        z = near[..., None] * (1. - t_vals) + far[..., None] * t_vals
        if t_rand is not None:
            mids = .5 * (z[..., 1:] + z[..., :-1])
            upper = torch.cat([mids, z[..., -1:]], -1)
            lower = torch.cat([z[..., :1], mids], -1)
            z = lower + (upper - lower) * t_rand.to(device=dev, dtype=torch.float32)
        return z

    def render_rays_hierarchical(self, ray_o, ray_d, near, far, feature_volume, sp_input, t_rand=None, u=None):
        """Coarse pass (cfg.N_samples) -> importance samples from its weights -> fine pass over the merged depths with the SAME
        network, as the reference's NeRF-baseline renderer does (volume_renderer.py:60-118; Neural Body's own renderer has no
        fine pass, SURVEY 8f-4).  `cfg.render_importance` = N_importance; det = (cfg.perturb == 0) as upstream.
        Both passes are nb_render_fwd launches (the fine one with nb_render_args.z_vals); under autograd each is a
        `_FusedRender` node and the importance samples are detached, as upstream."""
        cfg = get_active_cfg()
        Ni = int(self._opt("render_importance", 0))
        S = int(cfg.N_samples)
        dev = ray_o.device
        B, n = int(ray_o.shape[0]), int(ray_o.shape[1])
        if t_rand is None and float(cfg.perturb) > 0. and self.net.training:
            t_rand = self._draw_t_rand(B, n, S, dev)
        if u is None and float(cfg.perturb) != 0.:
            u = torch.rand((B * n, Ni)).view(B, n, Ni).to(dev)          # nerf_net_utils.py:70 (CPU generator, like upstream)
        coarse = self.render_rays(ray_o, ray_d, near, far, feature_volume, sp_input, t_rand=t_rand,
                                  want_weights=True)          # the coarse weights drive the importance sampling
        z_all, z_smp = self.importance_z_vals(near, far, coarse['weights'], S, Ni, t_rand=t_rand, u=u)
        fine = dict(self.render_rays(ray_o, ray_d, near, far, feature_volume, sp_input, z_vals=z_all))
        fine['rgb0'], fine['disp0'], fine['acc0'] = coarse['rgb_map'], coarse['disp_map'], coarse['acc_map']
        fine['z_std'] = torch.std(z_smp, dim=-1, unbiased=False)
        return fine

    # ------------------------------------------------------------------ the demo datasets' camera
    def camera_rays(self, batch):
        """The rays of a batch that carries the render camera instead of them (this package's multi_view_demo_dataset,
        multi_view_perform_dataset and monocular_demo_dataset drop-ins: `cam_RT`, `cam_K`, `can_bounds`), generated on the
        device as upstream's render_utils.image_rays generates them on the host, bit for bit (neuralbody_b200.rays.
        camera_image_rays; a float64 camera runs nb_image_rays_f64, a float32 one nb_image_rays, a mixed one is a
        ValueError).  The camera is read from batch['meta'] when it is there: upstream's visualize loop (run.py) moves every
        key but 'meta' to the GPU, and the drop-ins put a copy of the camera there, so reading it costs no device copy and
        the view's one host synchronisation is reading n.  Without it the camera keys are copied to the host in one
        transfer.  Sets batch['mask_at_box'] (1, H*W) bool on the device, which upstream's visualizers read; returns
        ray_o, ray_d (1,n,3), near, far (1,n)."""
        from neuralbody_b200 import rays
        cfg = get_active_cfg()
        keys = ('cam_RT', 'cam_K', 'can_bounds')
        meta = batch.get('meta')
        if isinstance(meta, dict) and 'train_cam' in meta and ('img' in batch or 'img_u8' in batch):   # the training
            # datasets' test split
            return self._dataset_view_rays(batch, meta)
        src = meta if isinstance(meta, dict) and all(k in meta for k in keys) else batch
        if any(src[k].shape[0] != 1 for k in keys):
            raise ValueError("a camera batch renders one view (batch size 1, as upstream's demo loaders)")
        H, W = cfg.H * cfg.ratio, cfg.W * cfg.ratio
        if H != int(H) or W != int(W):
            raise ValueError("cfg.H * cfg.ratio and cfg.W * cfg.ratio must be whole pixels (got %s x %s)" % (H, W))
        dev = batch['coord'].device if batch['coord'].device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        ray_o, ray_d, near, far, mask = rays.camera_image_rays(src['cam_RT'][0], src['cam_K'][0], src['can_bounds'][0],
                                                               int(H), int(W), device=dev)
        batch['mask_at_box'] = mask[None]
        return ray_o[None], ray_d[None], near[None], far[None]

    def _dataset_view_rays(self, batch, meta):
        """camera_rays for the training datasets' test split (multi_view_dataset / monocular_dataset drop-ins): `img`
        (1,H,W,3) and meta['train_cam'] / ['train_k_kind'] -> upstream's sample_ray(_h36m) test-split rays, bit for bit
        (rays.dataset_image_rays); also sets batch['rgb'] (1,n,3) and batch['mask_at_box'] (1,H*W) on the device."""
        from neuralbody_b200 import rays
        if 'img' not in batch:
            self.item_images(batch)
        img = batch['img']
        if img.shape[0] != 1:
            raise ValueError("a test-split batch renders one view (batch size 1, as upstream's test loader)")
        dev = img.device if img.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        H, W = int(img.shape[1]), int(img.shape[2])
        ray_o, ray_d, near, far, mask, rgb = rays.dataset_image_rays(torch.as_tensor(meta['train_cam'])[0].numpy(),
                                                                     int(torch.as_tensor(meta['train_k_kind']).reshape(-1)[0]),
                                                                     H, W, img[0].to(dev), device=dev)
        batch['mask_at_box'] = mask[None]
        batch['rgb'] = rgb[None]
        return ray_o[None], ray_d[None], near[None], far[None]

    # ------------------------------------------------------------------ the training datasets' sampled rays
    def train_rays(self, batch, draws=None):
        """The rays of a training batch that carries the image instead of them (this package's multi_view_dataset and
        monocular_dataset drop-ins, split 'train': `img` (B,H,W,3) float32, `ray_class` (B,H,W) uint8 and, in batch['meta']
        on the host, `train_cam` (B, NB_TRAIN_CAM_DOUBLES), `train_k_kind`, `N_rand`, `body_sample_ratio` and
        `face_sample_ratio`).  Draws N_rand pixels per item on the device as upstream's sample_ray_h36m / sample_ray do on
        the host (neuralbody_b200.rays.train_rays; `draws`: upstream's recorded np.random.randint results, for tests) and
        writes upstream's keys into the batch: ray_o, ray_d, rgb (B,N_rand,3), near, far (B,N_rand) float32 and an all-True
        mask_at_box (B,N_rand) bool, on the image's device.  Nothing synchronises with the host: the sampler's status is
        checked by the next render() after its prepare_sp_input, or by `check_train_rays()`.  A loop that refines cameras
        calls this first and then edits the rays; they are constants, as upstream's are."""
        from neuralbody_b200 import rays
        meta = batch['meta']
        if 'ray_class' not in batch:
            self.item_images(batch)
        img, cmap = batch['img'], batch['ray_class']
        if img.device.type != "cuda":
            dev = torch.device("cuda", torch.cuda.current_device())
            img, cmap = img.to(dev, non_blocking=True), cmap.to(dev, non_blocking=True)
        same = {}
        for k in ('train_k_kind', 'N_rand', 'body_sample_ratio', 'face_sample_ratio'):
            vals = set(torch.as_tensor(meta[k]).reshape(-1).tolist())
            if len(vals) != 1:
                raise ValueError("a training batch's items must share %s (got %s)" % (k, sorted(vals)))
            same[k] = vals.pop()
        res = rays.train_rays(img, cmap, torch.as_tensor(meta['train_cam']).numpy(), int(same['train_k_kind']),
                              int(same['N_rand']), float(same['body_sample_ratio']), float(same['face_sample_ratio']),
                              draws=draws)
        batch.update({'ray_o': res.ray_o, 'ray_d': res.ray_d, 'near': res.near, 'far': res.far, 'rgb': res.rgb,
                      'mask_at_box': torch.ones(tuple(res.near.shape), dtype=torch.bool, device=res.near.device)})
        self._train_rays_pending = res
        return res

    def item_images(self, batch):
        """The image steps of a batch from the training datasets' `dataset_image_steps: 'device'` items (`img_u8`
        (B,H0,W0,3), `msk_u8` (B,H0,W0) uint8, split 'train' also `bound_mask` (B,H,W), and in batch['meta'] on the host
        `image_cam`, `image_n_dist`, `image_size`, `image_bkgd`, `image_class`, `image_msk`): undistort, resize, background
        and class map on the device (neuralbody_b200.images.item_images, bit for bit with the host item's cv2 steps).  Writes
        `img` (B,H,W,3) float32, for split 'train' `ray_class` (B,H,W) uint8, and for People-Snapshot `msk` (B,H,W) uint8
        into the batch.  Raises ValueError when the items differ in size or steps.  Nothing synchronises with the host."""
        from neuralbody_b200 import images
        meta = batch['meta']
        img_u8, msk_u8 = batch['img_u8'], batch['msk_u8']
        dev = img_u8.device if img_u8.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        same = {}
        for k in ('image_n_dist', 'image_bkgd', 'image_class', 'image_msk'):
            vals = set(torch.as_tensor(meta[k]).reshape(-1).tolist())
            if len(vals) != 1:
                raise ValueError("a batch's items must share %s (got %s)" % (k, sorted(vals)))
            same[k] = int(vals.pop())
        sizes = set(map(tuple, torch.as_tensor(meta['image_size']).reshape(-1, 2).tolist()))
        if len(sizes) != 1:
            raise ValueError("a batch's items must share the image size (got %s)" % sorted(sizes))
        H, W = sizes.pop()
        bound = batch['bound_mask'] if same['image_class'] else None
        img, msk, cmap = images.item_images(img_u8.to(dev, non_blocking=True), msk_u8.to(dev, non_blocking=True),
                                            torch.as_tensor(meta['image_cam']).reshape(-1, images.capi.NB_ITEM_CAM_DOUBLES).numpy(),
                                            same['image_n_dist'], H, W, same['image_bkgd'], same['image_class'], bound)
        batch['img'] = img
        if cmap is not None:
            batch['ray_class'] = cmap
        if same['image_msk']:
            batch['msk'] = msk
        return batch

    # the batch key mask_views writes: upstream's masked renderers read the views as `msks` (1,nv,H,W); the single-view
    # renderer (if_nerf_renderer_msk) reads `msk` (1,H,W)
    MASK_VIEWS_KEY = 'msks'

    def mask_views(self, batch):
        """The mask steps of a batch from the demo and mesh datasets' `dataset_image_steps: 'device'` items (`msks_u8`
        (1,nv,H0,W0) uint8 as decoded, and in batch['meta'] on the host `mask_cams`, `mask_n_dist`, `mask_size`,
        `mask_binarise`, `mask_dilate`): binarise, undistort, dilate and resize on the device (neuralbody_b200.images.
        mask_views, bit for bit with upstream's cv2 steps).  Writes `msks` (1,nv,H,W) uint8 into the batch, or `msk` (1,H,W)
        for the single-view renderer (MASK_VIEWS_KEY).  B = 1, as upstream's loaders.  Nothing synchronises with the host."""
        from neuralbody_b200 import images
        meta, msk_u8 = batch['meta'], batch['msks_u8']
        if msk_u8.dim() != 4 or msk_u8.shape[0] != 1:
            raise ValueError("batch['msks_u8'] must be (1,nv,H0,W0) (B = 1, as upstream); got %s" % (tuple(msk_u8.shape),))
        if self.MASK_VIEWS_KEY == 'msk' and msk_u8.shape[1] != 1:
            raise ValueError("the single-view renderer takes one mask view (got %d)" % msk_u8.shape[1])
        dev = msk_u8.device if msk_u8.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())
        one = lambda k: int(torch.as_tensor(meta[k]).reshape(-1)[0])
        H, W = (int(v) for v in torch.as_tensor(meta['mask_size']).reshape(-1)[:2])
        cams = torch.as_tensor(meta['mask_cams']).reshape(-1, images.capi.NB_ITEM_CAM_DOUBLES).numpy()
        out = images.mask_views(msk_u8[0].to(dev, non_blocking=True), cams, one('mask_n_dist'), H, W,
                                one('mask_binarise'), one('mask_dilate'))
        batch[self.MASK_VIEWS_KEY] = out[None] if self.MASK_VIEWS_KEY == 'msks' else out
        return batch

    def check_train_rays(self):
        """Raise RuntimeError when the last train_rays call failed (a view whose bound pixels' rays all miss the box, where
        upstream loops forever)."""
        res = self.__dict__.pop("_train_rays_pending", None)
        if res is not None:
            res.check()

    # ------------------------------------------------------------------ a1
    def render(self, batch):
        """if_clight_renderer.py:94-122.  `cfg.chunk` rays per launch (0 = everything in one
        launch; upstream hard-codes 2048 to bound activation memory, which the fused kernel
        never materialises).  A batch without `ray_o` but with the render camera (`cam_RT`, `cam_K`, `can_bounds`) gets
        its rays from `camera_rays`; a training batch without `ray_o` but with the image (`img`, `ray_class`, or the
        decoded `img_u8` with `bound_mask`, which `item_images` processes first) gets them from `train_rays`, issued before
        prepare_sp_input's host synchronisation and checked after it; a test-split batch of those datasets (`img` or
        `img_u8` without a class map) gets the whole view's rays and colours from `camera_rays`."""
        if 'ray_o' not in batch and ('ray_class' in batch or 'bound_mask' in batch):
            self.train_rays(batch)
        if 'ray_o' not in batch and ('cam_RT' in batch or 'img' in batch or 'img_u8' in batch):
            ray_o, ray_d, near, far = self.camera_rays(batch)
        else:
            ray_o = batch['ray_o']
            ray_d = batch['ray_d']
            near = batch['near']
            far = batch['far']

        sp_input = self.prepare_sp_input(batch)
        self.check_train_rays()   # after the .tolist() above waited for the stream: no second synchronisation
        feature_volume = self.net.encode_sparse_voxels(sp_input)

        n_pixel = ray_o.shape[1]
        chunk = int(self._opt("chunk", 0)) or n_pixel
        if chunk >= n_pixel:
            return self.get_pixel_value(ray_o, ray_d, near, far, feature_volume, sp_input, batch)
        ret_list = []
        for i in range(0, n_pixel, chunk):
            ret_list.append(self.get_pixel_value(ray_o[:, i:i + chunk], ray_d[:, i:i + chunk], near[:, i:i + chunk],
                                                 far[:, i:i + chunk], feature_volume, sp_input, batch))
        keys = ret_list[0].keys()
        return {k: torch.cat([r[k] for r in ret_list], dim=1) for k in keys}
