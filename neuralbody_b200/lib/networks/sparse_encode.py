"""f-2(ii): dense-PyTorch emulation of the reference's SparseConvNet encode (lib/networks/latent_xyzc.py:30-39,166-274),
for machines without spconv -- OPT-IN (`Network.attach_dense_encoder()` or `sparse_encode: 'dense'`); by default the encode
stays on the reference's spconv path and this package's hot path starts at the four dense volumes it returns.  The same
encode runs as sparse convolutions on the GPU in CudaSparseConvNet (sparse_encode_cuda.py, `sparse_encode: 'cuda'`,
also opt-in), which is tested against this module in float64.

PARITY UNPINNED: spconv 1.2.1 (commit abf0acf, INSTALL.md:14-22) is not in this image, so this module cannot be checked
against it.  It follows spconv's published semantics, restated independently as a brute-force sparse oracle in
oracle/spconv_oracle.py (tests/test_sparse_encode.py compares the two):
  * SubMConv3d(k=3, bias=False): outputs only at the input-active sites; each is the cross-correlation over its ACTIVE
    neighbours, weight layout [kD, kH, kW, Cin, Cout];
  * SparseConv3d(k=3, s=2, p=1, bias=False): output size floor((in - 1) / 2) + 1 per axis, a site is active iff any input
    in its 3x3x3 window is active;
  * BatchNorm1d(eps=1e-3, momentum=0.01) over the ACTIVE rows only (batch statistics in train mode -- upstream renders
    with network.train(), run.py:57,89), then ReLU;
  * .dense(): (B, C, D, H, W), exact zeros off the active set;
  * several SMPL vertices falling into one 5 mm voxel are order-dependent upstream; here the highest vertex index wins.
Parameter names and shapes match the reference module tree (`conv0.0.weight` [3,3,3,16,16], `conv0.1.*` BatchNorm1d, ...), so a
reference checkpoint's `xyzc_net.*` entries load into this module unchanged.

Everything is plain dense torch ops on masked (B, C, D, H, W) tensors (137 MB x a few live tensors at the benchmark size);
the volumes are produced once per frame and cached across views by the renderer."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class _Conv(nn.Module):
    """One spconv convolution: weight [3,3,3,Cin,Cout] like spconv 1.2.1; `stride` 1 = SubMConv3d, 2 = SparseConv3d(p=1)."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        self.stride = stride
        w = torch.empty(3, 3, 3, cin, cout)
        nn.init.kaiming_uniform_(w.view(27 * cin, cout).t(), a=5 ** 0.5)      # spconv's reset_parameters
        self.weight = nn.Parameter(w)

    def forward(self, x, mask):
        w = self.weight.permute(4, 3, 0, 1, 2)                                 # -> conv3d's [Cout, Cin, kD, kH, kW]
        y = F.conv3d(x, w, stride=self.stride, padding=1)                     # x is exactly 0 off its active set
        if self.stride == 1:
            out_mask = mask                                                    # submanifold: the active set does not grow
        else:
            out_mask = F.max_pool3d(mask, 3, stride=2, padding=1)             # any active input in the window
        return y * out_mask, out_mask


def _masked_bn_relu(bn, x, mask):
    """BatchNorm1d over the active rows of a masked dense tensor, then ReLU; rows off the active set stay exactly 0."""
    C = x.shape[1]
    n = mask.sum().clamp_min(1.0)
    if bn.training or not bn.track_running_stats:
        mean = x.sum(dim=(0, 2, 3, 4)) / n
        var = (((x - mean.view(1, C, 1, 1, 1)) * mask) ** 2).sum(dim=(0, 2, 3, 4)) / n        # biased, as F.batch_norm normalises
        if bn.training and bn.track_running_stats:
            with torch.no_grad():
                m = bn.momentum
                bn.running_mean.mul_(1 - m).add_(m * mean)
                bn.running_var.mul_(1 - m).add_(m * var * n / (n - 1).clamp_min(1.0))          # unbiased in the running stats
                bn.num_batches_tracked += 1
    else:
        mean, var = bn.running_mean, bn.running_var
    y = (x - mean.view(1, C, 1, 1, 1)) * torch.rsqrt(var.view(1, C, 1, 1, 1) + bn.eps)
    y = y * bn.weight.view(1, C, 1, 1, 1) + bn.bias.view(1, C, 1, 1, 1)
    return F.relu(y) * mask


class _Block(nn.Sequential):
    """spconv.SparseSequential(conv, BatchNorm1d, ReLU, ...) with the reference's child indices (conv 0/3/6, bn 1/4/7)."""

    def __init__(self, cin, cout, n_convs, stride):
        layers = []
        for i in range(n_convs):
            layers += [_Conv(cin if i == 0 else cout, cout, stride), nn.BatchNorm1d(cout, eps=1e-3, momentum=0.01), nn.ReLU()]
        super().__init__(*layers)

    def forward(self, x, mask):
        for i in range(0, len(self), 3):
            x, mask = self[i](x, mask)
            x = _masked_bn_relu(self[i + 1], x, mask)
        return x, mask


class DenseSparseConvNet(nn.Module):
    """latent_xyzc.py:166-207 on masked dense tensors."""

    def __init__(self):
        super().__init__()
        self.conv0 = _Block(16, 16, 2, 1)      # double_conv 'subm0'
        self.down0 = _Block(16, 32, 1, 2)      # stride_conv 'down0'
        self.conv1 = _Block(32, 32, 2, 1)
        self.down1 = _Block(32, 64, 1, 2)
        self.conv2 = _Block(64, 64, 3, 1)      # triple_conv
        self.down2 = _Block(64, 128, 1, 2)
        self.conv3 = _Block(128, 128, 3, 1)
        self.down3 = _Block(128, 128, 1, 2)
        self.conv4 = _Block(128, 128, 3, 1)

    def forward(self, x, mask):
        """x (B,16,D,H,W) zero off `mask` (B,1,D,H,W) -> the four dense volumes [net1..net4] of latent_xyzc.py:181-207."""
        x, mask = self.conv0(x, mask)
        x, mask = self.down0(x, mask)
        x, mask = self.conv1(x, mask)
        net1 = x
        x, mask = self.down1(x, mask)
        x, mask = self.conv2(x, mask)
        net2 = x
        x, mask = self.down2(x, mask)
        x, mask = self.conv3(x, mask)
        net3 = x
        x, mask = self.down3(x, mask)
        x, mask = self.conv4(x, mask)
        return [net1, net2, net3, x]

    def encode(self, code, coord, out_sh, batch_size):
        """spconv.SparseConvTensor(code, coord, out_sh, batch_size) -> forward (latent_xyzc.py:35-37).
        code (6890,16) is shared by the frames of the batch; coord (B*6890,4) int = (frame, z, y, x)."""
        D, H, W = (int(v) for v in out_sh)
        B = int(batch_size)
        dev = code.device
        coord = coord.to(device=dev, dtype=torch.long)
        n_vert = code.shape[0]
        flat = ((coord[:, 0] * D + coord[:, 1]) * H + coord[:, 2]) * W + coord[:, 3]
        # duplicates (several vertices in one voxel): the highest vertex index wins, deterministically
        order = torch.arange(coord.shape[0], device=dev)
        winner = torch.full((B * D * H * W,), -1, dtype=torch.long, device=dev)
        winner = winner.scatter_reduce(0, flat, order, reduce="amax", include_self=True)
        active = winner >= 0
        feat = torch.zeros((B * D * H * W, code.shape[1]), dtype=code.dtype, device=dev)
        feat[active] = code[winner[active] % n_vert]
        x = feat.view(B, D, H, W, -1).permute(0, 4, 1, 2, 3).contiguous()
        mask = active.view(B, 1, D, H, W).to(code.dtype)
        return self.forward(x, mask)
