"""CPU: the drop-in boundary without a GPU -- the C-ABI library loads and exports every symbol
include/*.h declares, the config keeps the reference's key surface, the plugin factories pick
classes by file path, the Network keeps the reference's state_dict names, and the product path
refuses to run without CUDA (no silent fallback)."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT, golden_case


def _declared_functions():
    names = []
    inc = os.path.join(ROOT, "include")
    for fn in os.listdir(inc):
        if fn.endswith(".h"):
            src = open(os.path.join(inc, fn)).read()
            src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
            names += re.findall(r"\b(nb_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_library_exports_every_declared_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    declared = _declared_functions()
    assert len(declared) >= 9
    for name in declared:
        assert hasattr(lib, name), "include/neuralbody_b200.h declares %s but the library does not export it" % name
    from neuralbody_b200 import capi
    assert sorted(capi.EXPORTS) == declared
    assert capi.load().nb_abi_version() == 6


def test_struct_layouts_match_header(built_lib):
    """ctypes mirrors must have the C sizes (compile a probe with gcc against the header)."""
    import subprocess
    import tempfile
    from neuralbody_b200 import capi
    src = ('#include <stdio.h>\n#include "neuralbody_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(nb_volume_level), '
           'sizeof(nb_decoder_weights), sizeof(nb_render_args), sizeof(nb_importance_args), sizeof(nb_image_rays_args));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "p")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(capi.nb_volume_level), ctypes.sizeof(capi.nb_decoder_weights),
                     ctypes.sizeof(capi.nb_render_args), ctypes.sizeof(capi.nb_importance_args),
                     ctypes.sizeof(capi.nb_image_rays_args)]


def test_size_queries_without_gpu(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    dims = capi.LevelDims()
    for l, (c, d, h, w) in enumerate([(32, 48, 176, 96), (64, 24, 88, 48), (128, 12, 44, 24), (128, 6, 22, 12)]):
        dims[l][0], dims[l][1], dims[l][2], dims[l][3] = c, d, h, w
    n32 = lib.nb_packed_volume_bytes(dims, 1, capi.NB_DTYPE_F32)
    n16 = lib.nb_packed_volume_bytes(dims, 1, capi.NB_DTYPE_F16)
    # SURVEY 8a: 137 MB fp32 / 69 MB fp16 of features (+ ~0.3 MB of occupancy bitmaps in both)
    assert n32 >= 137 * 10 ** 6 and abs((n32 - n16) - 68530176) < 4096 and n16 < 70 * 10 ** 6
    assert lib.nb_packed_volume_level_offset(dims, 1, capi.NB_DTYPE_F16, 0) == 0
    assert lib.nb_packed_weights_bytes(2) > lib.nb_packed_weights_bytes(1) > 15 * 10 ** 5
    # argument validation happens before any CUDA call
    assert lib.nb_render_fwd(None, None) < 0
    assert b"null" in lib.nb_last_error()
    # scratch of the tensor-core pipeline: a 32-byte control block per frame + 3 x 16 B per sample of ONE frame
    # (two list buffers, each shared by two sample classes, + the raw records)
    ws = lib.nb_render_fwd_workspace_bytes
    per_frame = 512 * 512 * 64 * 16
    assert ws(1, 512 * 512, 64) == 256 + 3 * per_frame and ws(3, 512 * 512, 64) == ws(1, 512 * 512, 64)
    assert ws(0, 10, 10) == 0 and ws(1, 1000, 192) >= 2 * 1000 * 192 * 16
    # f-4: nb_sample_pdf validates its sizes before it touches the device
    a = capi.nb_importance_args()
    a.n_rays_total, a.n_samples, a.n_importance = 10, 2, 8
    assert lib.nb_sample_pdf(ctypes.byref(a), None) < 0 and b"n_samples >= 3" in lib.nb_last_error()
    a.n_samples, a.n_importance = 300, 8
    assert lib.nb_sample_pdf(ctypes.byref(a), None) < 0 and b"supported" in lib.nb_last_error()
    a.n_samples, a.n_importance = 64, 128
    assert lib.nb_sample_pdf(ctypes.byref(a), None) < 0 and b"null" in lib.nb_last_error()


def test_training_buffer_pool_is_best_fit():
    """The renderer recycles the activation record / backward scratch (host logic, device-agnostic): a small request must not
    take the large buffer a later, larger request needs (coarse vs fine pass of a hierarchical step)."""
    from neuralbody_b200.lib.networks.renderer.if_nerf_renderer import Renderer
    r = Renderer.__new__(Renderer)
    big = r._pool_take("save", 3000, torch.float32, torch.device("cpu"))
    small = r._pool_take("save", 1000, torch.float32, torch.device("cpu"))
    r._pool_give("save", big)
    r._pool_give("save", small)
    assert r._pool_take("save", 900, torch.float32, torch.device("cpu")) is small
    assert r._pool_take("save", 2500, torch.float32, torch.device("cpu")) is big
    fresh = r._pool_take("save", 10, torch.float32, torch.device("cpu"))
    assert fresh is not small and fresh is not big and fresh.numel() == 10


def test_config_surface_and_overrides(tmp_path):
    from neuralbody_b200.lib.config import CfgNode, make_cfg
    from neuralbody_b200.lib.config.config import _defaults
    c = _defaults()
    for key in ("N_samples", "perturb", "raw_noise_std", "white_bkgd", "voxel_size", "xyz_res", "view_res",
                "num_train_frame", "H", "W", "ratio", "renderer_module", "renderer_path", "network_module",
                "network_path", "N_rand"):
        assert key in c, key
    here = os.path.join(ROOT, "neuralbody_b200", "configs", "synth_snapshot_f3c.yaml")
    make_cfg(here, ["N_samples", "128", "white_bkgd", "True", "train.lr", "5e-4"], target=c)
    assert c.num_train_frame == 230 and c.H == 1080          # child overrides parent_cfg
    assert c.N_samples == 128 and c.white_bkgd is True and c.train.lr == 5e-4
    assert c.voxel_size == [0.005, 0.005, 0.005]             # inherited from parent
    with pytest.raises(ValueError):
        c.merge_from_list(["dangling"])


def test_factories_and_state_dict_compat(built_lib):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks import make_network
    from neuralbody_b200.lib.networks.renderer import make_renderer
    scene, _, _ = golden_case("eval_s64")
    cfg.num_train_frame = 60
    net = make_network(cfg)
    sd = net.state_dict()
    expect = {"c.weight": (6890, 16), "latent.weight": (60, 128), "fc_0.weight": (256, 352, 1), "fc_0.bias": (256,),
              "fc_1.weight": (256, 256, 1), "fc_2.weight": (256, 256, 1), "alpha_fc.weight": (1, 256, 1),
              "feature_fc.weight": (256, 256, 1), "latent_fc.weight": (256, 384, 1), "view_fc.weight": (128, 346, 1),
              "rgb_fc.weight": (3, 128, 1), "rgb_fc.bias": (3,)}
    for k, shp in expect.items():
        assert tuple(sd[k].shape) == shp, k
    missing, unexpected = net.load_state_dict(scene["weights"], strict=False)
    assert not unexpected and set(missing) == {"c.weight"}
    ren = make_renderer(cfg, net)
    assert type(ren).__name__ == "Renderer" and ren.net is net
    for m in ("render", "get_pixel_value", "get_sampling_points", "prepare_sp_input", "get_density_color"):
        assert callable(getattr(ren, m))
    # prepare_sp_input keeps upstream semantics (if_clight_renderer.py:29-52)
    sp = ren.prepare_sp_input({k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")})
    assert sp["coord"].shape == (6890, 4) and sp["out_sh"] == scene["out_sh"][0].tolist() and sp["batch_size"] == 1
    # host-side get_sampling_points agrees with the oracle restatement
    from oracle import neuralbody_oracle as O
    cfg.N_samples, cfg.perturb = 64, 0.0
    p1, z1 = ren.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"])
    p2, z2 = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], 64)
    assert torch.equal(p1, p2) and torch.equal(z1, z2)


def test_no_cpu_fallback(built_lib):
    """The render path must fail loudly without CUDA tensors / without the extension."""
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks import make_network
    from neuralbody_b200.lib.networks.renderer import make_renderer
    scene, _, _ = golden_case("eval_s64")
    cfg.num_train_frame = 60
    net = make_network(cfg)
    net.set_feature_volume(scene["volumes"])
    ren = make_renderer(cfg, net)
    batch = {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index", "ray_o", "ray_d", "near", "far")}
    with pytest.raises(RuntimeError, match="CUDA"):
        ren.render(batch)
    with pytest.raises(RuntimeError, match="not found"):
        capi.load("/nonexistent/libneuralbody_b200.so")
    net.set_feature_volume(None)
    with pytest.raises(RuntimeError, match="reference"):
        net.encode_sparse_voxels({})
