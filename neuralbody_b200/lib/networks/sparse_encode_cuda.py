"""The reference's SparseConvNet encode (lib/networks/latent_xyzc.py:30-39,166-274) on the GPU as sparse convolutions:
nb_spconv_fwd / nb_spconv_bwd (csrc/nb_spconv.cu), opt-in with `sparse_encode: 'cuda'` or `Network.attach_cuda_encoder()`.

`CudaSparseConvNet` has the parameter tree of `DenseSparseConvNet` (sparse_encode.py), i.e. the reference module's, so a
reference checkpoint's `xyzc_net.*` entries and the emulation's state dict load into it unchanged.  Its `encode` computes
what `DenseSparseConvNet.encode` computes -- the semantics listed in sparse_encode.py's header, the same duplicate rule, four
dense NCDHW fp32 volumes with exact zeros off the active set -- but convolves the active sites only, in fp32 FFMA with
float64 BatchNorm sums.  Train mode normalises with the batch statistics and updates running_mean / running_var /
num_batches_tracked; eval mode uses the running statistics.  Gradients reach `code` (so `c.weight`), every conv weight and
every BatchNorm weight and bias.  Nothing waits for the host: the row buffers are sized from bounds, and the row counts stay
on the device (`last_row_counts`, int32 [5]: active sites of the input grid and of the four levels)."""
import ctypes as C

import torch

from neuralbody_b200 import capi
from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet

_BLOCKS = ("conv0", "down0", "conv1", "down1", "conv2", "down2", "conv3", "down3", "conv4")


def _check_float(name, t, dev):
    if not torch.is_tensor(t) or t.dtype != torch.float32 or t.device != dev:
        raise ValueError("%s must be a float32 tensor on %s (got %s)" % (
            name, dev, "%s %s" % (t.dtype, t.device) if torch.is_tensor(t) else type(t).__name__))


class _Encode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, coord, out_sh, batch_size, code, *params):
        L = capi.NB_SPCONV_LAYERS
        dev = code.device
        bns = net.batchnorms()
        a = capi.nb_spconv_args()
        a.batch, a.n_points, a.n_vert = batch_size, coord.shape[0], code.shape[0]
        for i in range(3):
            a.out_sh[i] = out_sh[i]
        code = code.detach().contiguous()
        params = [p.detach().contiguous() for p in params]
        a.coord, a.code = coord.data_ptr(), code.data_ptr()
        for j in range(L):
            a.weight[j], a.bn_weight[j], a.bn_bias[j] = (params[j].data_ptr(), params[L + j].data_ptr(),
                                                         params[2 * L + j].data_ptr())
            a.running_mean[j], a.running_var[j] = bns[j].running_mean.data_ptr(), bns[j].running_var.data_ptr()
            a.num_batches_tracked[j] = bns[j].num_batches_tracked.data_ptr()
        a.training = 1 if net.training else 0
        a.momentum, a.eps = bns[0].momentum, bns[0].eps
        lib = capi.load()
        ws = torch.empty(lib.nb_spconv_workspace_bytes(a.batch, a.n_points, a.out_sh), dtype=torch.uint8, device=dev)
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
        vols = [torch.empty((batch_size, c) + s, dtype=torch.float32, device=dev)
                for c, s in zip((32, 64, 128, 128), level_shapes(out_sh))]
        for l, v in enumerate(vols):
            a.volumes[l] = v.data_ptr()
        counts = torch.empty(5, dtype=torch.int32, device=dev)
        a.row_counts = counts.data_ptr()
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(lib.nb_spconv_fwd(C.byref(a), C.c_void_p(stream)), "nb_spconv_fwd")
        net.last_row_counts = counts
        # the workspace holds what the backward reads; the tensors behind a's pointers stay alive with it
        ctx.args, ctx.keep = a, (ws, coord, code, params)
        ctx.set_materialize_grads(False)
        return tuple(vols)

    @staticmethod
    def backward(ctx, *d_vols):
        L = capi.NB_SPCONV_LAYERS
        a = ctx.args
        ws, coord, code, params = ctx.keep
        dev = code.device
        g = capi.nb_spconv_grads()
        keep = []
        for l, d in enumerate(d_vols):
            if d is not None:
                d = d.to(dtype=torch.float32).contiguous()
                keep.append(d)
                g.d_volumes[l] = d.data_ptr()
        d_code = torch.empty_like(code)
        d_params = [torch.empty_like(p) for p in params]
        g.d_code = d_code.data_ptr()
        for j in range(L):
            g.d_weight[j], g.d_bn_weight[j], g.d_bn_bias[j] = (d_params[j].data_ptr(), d_params[L + j].data_ptr(),
                                                               d_params[2 * L + j].data_ptr())
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            capi.check(capi.load().nb_spconv_bwd(C.byref(a), C.byref(g), C.c_void_p(stream)), "nb_spconv_bwd")
        return (None, None, None, None, d_code) + tuple(d_params)


def level_shapes(out_sh):
    """(D, H, W) of the four strided levels: floor((in - 1) / 2) + 1 per axis, each from the previous one."""
    shapes, cur = [], [int(v) for v in out_sh]
    for _ in range(4):
        cur = [(v - 1) // 2 + 1 for v in cur]
        shapes.append(tuple(cur))
    return shapes


class CudaSparseConvNet(DenseSparseConvNet):
    """latent_xyzc.py:166-207 on the GPU's sparse convolutions; the parameter tree is DenseSparseConvNet's."""

    def __init__(self):
        super().__init__()
        self.last_row_counts = None

    def convs_and_batchnorms(self):
        """The 17 (conv, BatchNorm1d) pairs in the network's order."""
        out = []
        for name in _BLOCKS:
            blk = getattr(self, name)
            out += [(blk[i], blk[i + 1]) for i in range(0, len(blk), 3)]
        return out

    def batchnorms(self):
        return [bn for _, bn in self.convs_and_batchnorms()]

    def forward(self, code, coord, out_sh, batch_size):
        return self.encode(code, coord, out_sh, batch_size)

    def encode(self, code, coord, out_sh, batch_size):
        """spconv.SparseConvTensor(code, coord, out_sh, batch_size) -> [net1..net4] (latent_xyzc.py:35-37).  code (n_vert,16)
        float32 on a CUDA device is shared by the frames of the batch; coord (n_points,4) int = (frame, z, y, x), point i
        takes code[i % n_vert]; out_sh = (D, H, W)."""
        dev = code.device
        if dev.type != "cuda":
            raise ValueError("CudaSparseConvNet.encode runs on a CUDA device (code is on %s)" % dev)
        _check_float("code", code, dev)
        if code.dim() != 2 or code.shape[1] != 16:
            raise ValueError("code must be (n_vert, 16) (got %s)" % (tuple(code.shape),))
        if not torch.is_tensor(coord) or coord.dim() != 2 or coord.shape[1] != 4 or coord.is_floating_point():
            raise ValueError("coord must be an (n_points, 4) integer tensor")
        pairs = self.convs_and_batchnorms()
        params = [c.weight for c, _ in pairs] + [bn.weight for _, bn in pairs] + [bn.bias for _, bn in pairs]
        for i, p in enumerate(params):
            _check_float("parameter %d" % i, p, dev)
        for _, bn in pairs:
            if bn.momentum is None or not bn.track_running_stats or bn.momentum != pairs[0][1].momentum \
                    or bn.eps != pairs[0][1].eps:
                raise ValueError("every BatchNorm1d needs running statistics and the same momentum (not None) and eps")
            _check_float("running stats", bn.running_mean, dev)
            _check_float("running stats", bn.running_var, dev)
        out_sh = [int(v) for v in out_sh]
        coord = coord.to(device=dev, dtype=torch.int32).contiguous()
        return list(_Encode.apply(self, coord, out_sh, int(batch_size), code, *params))
