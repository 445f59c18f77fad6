"""GPU: density queries on the tensor cores (cfg.density_precision 'tc_fp16x3' / 'tc_fp16', nb_decode_density_list) against
the oracle's Network.calculate_density, exact empty-point skipping, independence of the tile a point lands in, the mesh
renderer on them, and the calls the C ABI refuses."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import golden_case
from oracle import mcubes_oracle as M
from oracle import mesh_case
from oracle import neuralbody_oracle as O
import gpu_utils as G
from neuralbody_b200 import capi
from neuralbody_b200.lib.config import cfg

pytestmark = pytest.mark.gpu


def _with(**kw):
    old = {k: (cfg[k] if k in cfg else None) for k in kw}
    for k, v in kw.items():
        cfg[k] = v
    return old


def _restore(old):
    for k, v in old.items():
        if v is None:
            if k in cfg:
                del cfg[k]
        else:
            cfg[k] = v


@pytest.fixture(scope="module")
def case():
    """The 2 x 5000 random points of test_density_only_decoder_matches_oracle (some outside the box) and the oracle's sigma."""
    scene, _, _ = golden_case("batch2_s32")
    net, ren = G.make_net_and_renderer(scene)
    g = torch.Generator().manual_seed(5)
    lo, hi = scene["can_bounds"][0, 0], scene["can_bounds"][0, 1]
    pts = (torch.rand((2, 5000, 3), generator=g) * 1.2 - 0.1) * (hi - lo) + lo
    want = O.calculate_density(scene["weights"], pts, scene["volumes"], O.prepare_sp_input(scene), scene["voxel_size"])
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    sp = ren.prepare_sp_input(batch)
    return net, ren, pts, want, sp, net.encode_sparse_voxels(sp)


def _density(case, precision, skip=True, pts=None, stats=None):
    net, ren, pts0, _, sp, fv = case
    old = _with(density_precision=precision, render_skip_empty=skip)
    try:
        ren.stats = stats
        out = ren.calculate_density((pts0 if pts is None else pts).cuda(), fv, sp)
        torch.cuda.synchronize()
    finally:
        _restore(old)
        ren.stats = None
    return out.cpu()


@pytest.mark.parametrize("precision,tol", [("tc_fp16x3", 5e-4), ("tc_fp16", 8e-2)])
def test_density_tc_matches_oracle(case, precision, tol):
    want = case[3]
    got = _density(case, precision)
    assert got.shape == want.shape == (2, 5000, 1)
    assert float((got - want).abs().max()) < tol
    assert float(want.max()) > 5.0 and float(want.min()) < -5.0          # not vacuous


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_density_tc_skipping_is_exact(case, precision):
    n = 2 * 5000
    s_on = torch.zeros(8, dtype=torch.int64, device="cuda")
    s_off = torch.zeros(8, dtype=torch.int64, device="cuda")
    on = _density(case, precision, skip=True, stats=s_on)
    off = _density(case, precision, skip=False, stats=s_off)
    listed = int(s_on[1])
    assert 0 < listed < n, listed
    assert int(s_off[1]) == n
    assert int(s_on[3]) == 2 and int(s_on[0]) > 0 and int(s_on[2]) > 0     # one decoder launch per frame, timed
    # the skipped points: exactly the blob's sigma(empty), one value, on n - listed points
    vals, counts = torch.unique(on, return_counts=True)
    top = vals[counts.argmax()]
    skipped = on == top
    assert int(skipped.sum()) >= n - listed
    # every point the decoder evaluated with skipping on has the same sigma bit for bit with skipping off
    ev = ~skipped
    assert torch.equal(on[ev].view(torch.int32), off[ev].view(torch.int32))
    # the skipped points are the ones with all-zero features: the dense run's decoder gives them (nearly) sigma(empty)
    assert float((off[skipped] - top).abs().max()) < (1e-3 if precision == "tc_fp16x3" else 1e-1)


def test_density_tc_skipped_value_is_sigma_empty(case):
    """sigma(empty) as the weight blob holds it: the decoder of a point with all-zero features, layers 0-2 and alpha_fc on
    the biases alone (exact fp32 in the blob); a skipped point gets exactly that value."""
    net = case[0]
    sd = {k: v.detach().double().cpu() for k, v in net.state_dict().items()}
    h = torch.relu(sd["fc_0.bias"])
    h = torch.relu(sd["fc_1.weight"].reshape(256, 256) @ h + sd["fc_1.bias"])
    h = torch.relu(sd["fc_2.weight"].reshape(256, 256) @ h + sd["fc_2.bias"])
    se = float(sd["alpha_fc.weight"].reshape(-1) @ h + sd["alpha_fc.bias"].reshape(-1)[0])
    on = _density(case, "tc_fp16x3")
    vals, counts = torch.unique(on, return_counts=True)
    top = float(vals[counts.argmax()])
    assert abs(top - se) < 1e-4, (top, se)


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_density_tc_permutation_invariant(case, precision):
    pts = case[2]
    perm = torch.randperm(pts.shape[1], generator=torch.Generator().manual_seed(11))
    a = _density(case, precision)
    b = _density(case, precision, pts=pts[:, perm])
    assert torch.equal(a[:, perm].view(torch.int32), b.view(torch.int32))


def _mesh_cube(case_name, precision):
    from test_mesh_gpu import _mesh_renderer, _render
    scene, _, batch = mesh_case.build_case(case_name)
    _, ren = _mesh_renderer(scene)
    old = _with(density_precision=precision)
    try:
        out = _render(ren, batch, 10.0)
    finally:
        _restore(old)
    return out


@pytest.mark.parametrize("case_name", ["mesh_s03", "mesh_full"])
def test_mesh_renderer_tc_fp16x3(case_name):
    ref = _mesh_cube(case_name, "fp32")
    out = _mesh_cube(case_name, "tc_fp16x3")
    cube, cref = out["cube"], ref["cube"]
    assert cube.shape == cref.shape
    assert float(np.abs(cube - cref).max()) < 5e-4
    if case_name == "mesh_s03":
        gold = mesh_case.load_golden()["cube"]
        assert (cube[gold == 0] == 0).all()
    assert (cube[cref == 0] == 0).all()                             # the scatter touches the inside points only
    vo, to = M.marching_cubes(cube.astype(np.float32), 10.0)
    f = np.asarray(out["mesh"].faces)
    np.testing.assert_array_equal(np.asarray(out["mesh"].vertices).view(np.int64), vo.view(np.int64))
    np.testing.assert_array_equal(f, to)
    assert len(f) > 2000 and M.closed_manifold_report(f)[0]
    nref = len(np.asarray(ref["mesh"].faces))
    assert abs(len(f) - nref) <= 0.01 * nref, (len(f), nref)


def test_density_list_rejections(case):
    net, ren, pts, _, sp, fv = case
    lib = capi.load()
    with torch.no_grad():
        ref = ren.calculate_density(pts.cuda(), fv, sp)          # fp32: a valid frame to start from
    torch.cuda.synchronize()
    vol_blob, dims = ren.pack_volume(fv, capi.NB_DTYPE_F32)
    w_blob = ren.pack_weights(sp["latent_index"], torch.device("cuda"))
    keep = [sp["R"].float().contiguous(), sp["Th"].float().reshape(2, 3).contiguous(), sp["bounds"].float().contiguous()]
    a = capi.nb_render_args()
    a.batch = 2
    a.R, a.Th, a.bounds = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr()
    for i in range(3):
        a.voxel_size[i] = float(cfg.voxel_size[i])
        a.out_sh[i] = int(sp["out_sh"][i])
    for l in range(capi.NB_NUM_LEVELS):
        for j in range(4):
            a.level_dims[l][j] = dims[l][j]
    a.volume_blob, a.volume_dtype, a.weights_blob = vol_blob.data_ptr(), capi.NB_DTYPE_F32, w_blob.data_ptr()
    stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    a.stats = stats.data_ptr()
    p = pts.cuda().contiguous()
    sigma = torch.full((2, 5000), 7.0, device="cuda")
    n = 5000
    ws = torch.empty(lib.nb_decode_density_workspace_bytes(2, n), dtype=torch.uint8, device="cuda")
    call = lambda k: lib.nb_decode_density_list(ctypes.byref(a), p.data_ptr(), k, sigma.data_ptr(), None)
    a.precision = capi.NB_PRECISION_FP32                                     # fp32 belongs to nb_decode_density
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    assert call(n) == -1 and b"nb_decode_density" in lib.nb_last_error()
    a.precision = capi.NB_PRECISION_TC_FP16X3
    a.workspace, a.workspace_bytes = None, 0                                 # missing workspace
    assert call(n) == -1 and b"workspace" in lib.nb_last_error()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel() - 1           # short workspace
    assert call(n) == -1 and b"workspace" in lib.nb_last_error()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    assert call(1 << 28) == -2 and b"2^28" in lib.nb_last_error()            # past the list's id range
    assert call(0) == 0                                                      # no-op
    torch.cuda.synchronize()
    assert bool((sigma == 7.0).all()) and int(stats.abs().sum()) == 0        # nothing was enqueued
    assert call(n) == 0                                                      # the same frame is accepted
    torch.cuda.synchronize()
    assert float((sigma.cpu() - ref[..., 0].cpu()).abs().max()) < 5e-4
