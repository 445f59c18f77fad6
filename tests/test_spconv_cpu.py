"""CPU: the sparse CUDA encoder's host side -- nb_spconv_fwd / nb_spconv_bwd refuse bad arguments before anything is
enqueued (the device pointers are placeholders, never dereferenced), the yaml key `sparse_encode` selects the encoder when
the network is built, and CudaSparseConvNet keeps the reference module's parameter tree."""
import ctypes
import json
import os

import pytest
import torch

from neuralbody_b200 import capi

NB_ERR_BAD_ARG = -1
FAKE = 0x10000
L = 17


def _args():
    """A call whose arguments all pass validation (the workspace size is the one the library asks for)."""
    a = capi.nb_spconv_args()
    a.batch, a.n_points, a.n_vert = 1, 6890, 6890
    for i, v in enumerate((96, 352, 192)):
        a.out_sh[i] = v
    a.coord = a.code = FAKE
    for j in range(L):
        a.weight[j] = a.bn_weight[j] = a.bn_bias[j] = a.running_mean[j] = a.running_var[j] = FAKE
        a.num_batches_tracked[j] = FAKE
    a.training, a.momentum, a.eps = 1, 0.01, 1e-3
    a.workspace = FAKE * 256
    a.workspace_bytes = capi.load().nb_spconv_workspace_bytes(a.batch, a.n_points, a.out_sh)
    for l in range(4):
        a.volumes[l] = FAKE
    return a


def _grads():
    g = capi.nb_spconv_grads()
    g.d_code = FAKE
    for j in range(L):
        g.d_weight[j] = g.d_bn_weight[j] = g.d_bn_bias[j] = FAKE
    return g


def _error():
    return capi.load().nb_last_error().decode()


DEFECTS = {
    "coord": lambda a: setattr(a, "coord", None),
    "code": lambda a: setattr(a, "code", None),
    "weight": lambda a: a.weight.__setitem__(9, None),
    "bn_bias": lambda a: a.bn_bias.__setitem__(16, None),
    "running_var": lambda a: a.running_var.__setitem__(3, None),
    "num_batches_tracked": lambda a: a.num_batches_tracked.__setitem__(0, None),
    "volumes": lambda a: a.volumes.__setitem__(2, None),
    "batch": lambda a: setattr(a, "batch", 0),
    "n_points": lambda a: setattr(a, "n_points", 0),
    "n_vert": lambda a: setattr(a, "n_vert", -1),
    "out_sh": lambda a: a.out_sh.__setitem__(1, 0),
    "training": lambda a: setattr(a, "training", 2),
    "eps": lambda a: setattr(a, "eps", 0.0),
    "momentum": lambda a: setattr(a, "momentum", 1.5),
    "workspace": lambda a: setattr(a, "workspace", None),
    "workspace_bytes": lambda a: setattr(a, "workspace_bytes", a.workspace_bytes - 1),
    "workspace_alignment": lambda a: setattr(a, "workspace", FAKE * 256 + 16),
}


@pytest.mark.parametrize("entry", ("nb_spconv_fwd", "nb_spconv_bwd"))
@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_bad_arguments_are_refused_under_the_entry_points_name(built_lib, entry, defect):
    a = _args()
    DEFECTS[defect](a)
    lib = capi.load()
    st = lib.nb_spconv_fwd(ctypes.byref(a), None) if entry == "nb_spconv_fwd" else \
        lib.nb_spconv_bwd(ctypes.byref(a), ctypes.byref(_grads()), None)
    assert st == NB_ERR_BAD_ARG
    assert _error().startswith(entry + ":"), _error()


def test_eval_mode_needs_no_num_batches_tracked(built_lib):
    """Only a training forward updates num_batches_tracked: in eval mode a NULL one passes validation (the call then fails
    on the next defect, here the workspace)."""
    a = _args()
    a.training = 0
    for j in range(L):
        a.num_batches_tracked[j] = None
    a.workspace = None
    assert capi.load().nb_spconv_fwd(ctypes.byref(a), None) == NB_ERR_BAD_ARG
    assert "workspace" in _error(), _error()


@pytest.mark.parametrize("defect", ("grads", "d_code", "d_weight", "d_bn_weight"))
def test_backward_refuses_missing_gradient_buffers(built_lib, defect):
    a, g = _args(), _grads()
    if defect == "d_code":
        g.d_code = None
    elif defect == "d_weight":
        g.d_weight[13] = None
    elif defect == "d_bn_weight":
        g.d_bn_weight[0] = None
    gp = None if defect == "grads" else ctypes.byref(g)
    assert capi.load().nb_spconv_bwd(ctypes.byref(a), gp, None) == NB_ERR_BAD_ARG
    assert _error().startswith("nb_spconv_bwd:") and "null" in _error(), _error()


def test_workspace_size_depends_on_the_sizes_only(built_lib):
    lib = capi.load()
    sh = (ctypes.c_int * 3)(96, 352, 192)
    one, two = lib.nb_spconv_workspace_bytes(1, 6890, sh), lib.nb_spconv_workspace_bytes(2, 2 * 6890, sh)
    assert 0 < one < two
    assert lib.nb_spconv_workspace_bytes(0, 6890, sh) == 0
    assert lib.nb_spconv_workspace_bytes(1, 6890, (ctypes.c_int * 3)(96, 0, 192)) == 0
    assert lib.nb_spconv_workspace_bytes(1024, 6890, (ctypes.c_int * 3)(1024, 1024, 1024)) == 0    # >= 2^31 sites


@pytest.fixture
def encoder_key():
    """The config the network reads when it is built: get_active_cfg(), i.e. upstream's cfg once the reference's lib.config
    is loaded in this process, else this package's.  sparse_encode is removed from it for one test and restored after."""
    from neuralbody_b200.lib.config import get_active_cfg
    cfg = get_active_cfg()
    had, old = "sparse_encode" in cfg, cfg.get("sparse_encode")
    dict.pop(cfg, "sparse_encode", None)

    def set_key(value):
        dict.__setitem__(cfg, "sparse_encode", value)      # dict's own setter: upstream's yacs node may be frozen
    yield set_key
    dict.pop(cfg, "sparse_encode", None)
    if had:
        dict.__setitem__(cfg, "sparse_encode", old)


@pytest.mark.parametrize("key,name", (("reference", "NoneType"), ("dense", "DenseSparseConvNet"), ("cuda", "CudaSparseConvNet")))
def test_yaml_key_selects_the_encoder(encoder_key, tmp_path, key, name):
    from neuralbody_b200.lib.config import CfgNode
    from neuralbody_b200.lib.networks.latent_xyzc import Network
    path = tmp_path / "enc.yaml"
    path.write_text("sparse_encode: '%s'\n" % key)
    parsed = CfgNode()
    parsed.merge_from_file(str(path))
    encoder_key(parsed.sparse_encode)
    net = Network(num_train_frame=4)
    assert type(net.xyzc_net).__name__ == name
    if key != "reference":
        assert {k for k in net.state_dict() if k.startswith("xyzc_net.")}


def test_default_is_the_reference_path_and_unknown_keys_raise(encoder_key):
    """A config without the key (upstream's) and this package's default both keep the reference path."""
    from neuralbody_b200.lib.config.config import _defaults
    from neuralbody_b200.lib.networks.latent_xyzc import Network
    assert _defaults().sparse_encode == "reference"
    assert Network(num_train_frame=4).xyzc_net is None
    encoder_key("spconv2")
    with pytest.raises(ValueError, match="sparse_encode"):
        Network(num_train_frame=4)


def test_reference_still_raises_without_a_spconv_module(encoder_key):
    from oracle import synth
    from neuralbody_b200.lib.networks.latent_xyzc import Network
    from neuralbody_b200.lib.networks.renderer.if_nerf_renderer import Renderer
    encoder_key("reference")
    scene = synth.make_scene(H=8, W=8, scale=0.12)
    net = Network(num_train_frame=4)
    ren = Renderer.__new__(Renderer)
    sp = Renderer.prepare_sp_input(ren, {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")})
    with pytest.raises(RuntimeError, match="SparseConvNet encode is outside this package"):
        net.encode_sparse_voxels(sp)


def test_parameter_tree_is_the_emulations_and_the_references():
    from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
    from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet
    dense, cuda = DenseSparseConvNet().state_dict(), CudaSparseConvNet().state_dict()
    assert list(dense) == list(cuda)
    assert all(dense[k].shape == cuda[k].shape and dense[k].dtype == cuda[k].dtype for k in dense)
    CudaSparseConvNet().load_state_dict(dense, strict=True)       # the emulation's state dict loads unchanged
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_sparseconvnet_bn_keys.json")) as f:
        ref_keys = set(json.load(f))
    assert ref_keys == {k for k in cuda if k.split(".")[1] in ("1", "4", "7")}
    assert len(CudaSparseConvNet().convs_and_batchnorms()) == L


def test_encode_refuses_cpu_tensors():
    """No fall-back: the encoder runs on the GPU or raises."""
    from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet
    with pytest.raises(ValueError, match="CUDA"):
        CudaSparseConvNet().encode(torch.zeros(6890, 16), torch.zeros(6890, 4, dtype=torch.int32), [8, 8, 8], 1)
