"""Network with the reference's parameter surface (lib/networks/latent_xyzc.py:9-28).

`state_dict()` keys and shapes of the decoder are identical to upstream
(`fc_0.weight (256,352,1)` ... `rgb_fc.weight (3,128,1)`, `latent.weight`, `c.weight`),
so reference checkpoints load with `load_state_dict(..., strict=False)`.

The SparseConvNet encode (`xyzc_net`, latent_xyzc.py:166-274) stays on the reference path by
default (SURVEY.md 8): attach the reference's own module as `net.xyzc_net` when spconv is
installed, or hand the dense volumes in with `set_feature_volume()` (what the synthetic scenes
do).  Two opt-in encoders need no spconv, selected by the yaml key `sparse_encode` when the
network is built ('reference' (default) | 'dense' | 'cuda') or from Python: the dense-PyTorch
emulation (`attach_dense_encoder()`, f-2(ii), parity unpinned) and the sparse CUDA
convolutions (`attach_cuda_encoder()`, csrc/nb_spconv.cu), both with the reference module's
parameter names.

The decoder arithmetic itself (`calculate_density_color`, :91-126) is not evaluated by
PyTorch modules here: the Renderer packs these parameters and runs the fused CUDA kernel.
"""
import torch
import torch.nn as nn

from neuralbody_b200.lib.config import get_active_cfg


class Network(nn.Module):
    def __init__(self, num_train_frame=None):
        super().__init__()
        cfg = get_active_cfg()
        if num_train_frame is None:
            num_train_frame = int(cfg.num_train_frame)
        self.c = nn.Embedding(6890, 16)
        self.xyzc_net = None                    # SparseConvNet stays on the reference path
        self.latent = nn.Embedding(num_train_frame, 128)
        self.actvn = nn.ReLU()
        self.fc_0 = nn.Conv1d(352, 256, 1)
        self.fc_1 = nn.Conv1d(256, 256, 1)
        self.fc_2 = nn.Conv1d(256, 256, 1)
        self.alpha_fc = nn.Conv1d(256, 1, 1)
        self.feature_fc = nn.Conv1d(256, 256, 1)
        self.latent_fc = nn.Conv1d(384, 256, 1)
        self.view_fc = nn.Conv1d(346, 128, 1)
        self.rgb_fc = nn.Conv1d(128, 3, 1)
        self._feature_volume = None
        encoder = cfg.get('sparse_encode', 'reference') if hasattr(cfg, 'get') else getattr(cfg, 'sparse_encode', 'reference')
        if encoder == 'dense':
            self.attach_dense_encoder()
        elif encoder == 'cuda':
            self.attach_cuda_encoder()
        elif encoder != 'reference':
            raise ValueError("sparse_encode must be 'reference', 'dense' or 'cuda' (got %r)" % (encoder,))

    # ---- encode: reference path or supplied volumes
    def set_feature_volume(self, volumes):
        """Supply the four dense NCDHW fp32 volumes `encode_sparse_voxels` should return."""
        self._feature_volume = None if volumes is None else list(volumes)

    def attach_dense_encoder(self):
        """f-2(ii), opt-in: run the encode with the dense-PyTorch emulation of the reference's SparseConvNet
        (lib/networks/sparse_encode.py; same parameter names, so `xyzc_net.*` of a reference checkpoint loads).  Parity
        against spconv is unpinned (spconv is absent from this image) -- see that module's header."""
        from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
        self.xyzc_net = DenseSparseConvNet().to(self.c.weight.device)
        return self.xyzc_net

    def attach_cuda_encoder(self):
        """Opt-in: run the encode as sparse convolutions on the GPU (lib/networks/sparse_encode_cuda.py, nb_spconv_fwd /
        nb_spconv_bwd), forward and backward; the same parameter names as the emulation and the reference module."""
        from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet
        self.xyzc_net = CudaSparseConvNet().to(self.c.weight.device)
        return self.xyzc_net

    def encode_sparse_voxels(self, sp_input):
        """latent_xyzc.py:30-39."""
        if self._feature_volume is not None:
            return self._feature_volume
        if type(self.xyzc_net).__name__ in ("DenseSparseConvNet", "CudaSparseConvNet"):
            coord = sp_input['coord']
            code = self.c(torch.arange(0, 6890).to(coord.device))
            return self.xyzc_net.encode(code, coord, sp_input['out_sh'], sp_input['batch_size'])
        if self.xyzc_net is None:
            raise RuntimeError(
                "SparseConvNet encode is outside this package (it stays on the reference's spconv path): "
                "attach the reference module as `net.xyzc_net` or call `net.set_feature_volume(volumes)`")
        import spconv  # reference path
        coord = sp_input['coord']
        code = self.c(torch.arange(0, 6890).to(coord.device))
        xyzc = spconv.SparseConvTensor(code, coord, sp_input['out_sh'], sp_input['batch_size'])
        return self.xyzc_net(xyzc)

    def calculate_density(self, wpts, feature_volume, sp_input):
        """latent_xyzc.py:74-89 (called by the reference's mesh renderer, if_mesh_renderer.py:36-39): (B,P,3) -> (B,P,1),
        evaluated by the fused density kernel (nb_decode_density); no PyTorch decoder path exists."""
        if getattr(self, "_density_renderer", None) is None:
            from neuralbody_b200.lib.networks.renderer.if_nerf_renderer import Renderer
            object.__setattr__(self, "_density_renderer", Renderer(self))
        return self._density_renderer.calculate_density(wpts, feature_volume, sp_input)

    def decoder_tensors(self):
        """The 17 decoder tensors in the order nb_decoder_weights expects."""
        return [self.fc_0.weight, self.fc_0.bias, self.fc_1.weight, self.fc_1.bias, self.fc_2.weight, self.fc_2.bias,
                self.alpha_fc.weight, self.alpha_fc.bias, self.feature_fc.weight, self.feature_fc.bias,
                self.latent_fc.weight, self.latent_fc.bias, self.view_fc.weight, self.view_fc.bias,
                self.rgb_fc.weight, self.rgb_fc.bias, self.latent.weight]
