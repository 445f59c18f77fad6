"""GPU: the sparse CUDA encoder (nb_spconv_fwd / nb_spconv_bwd) element by element against float64 on the edge cases of
oracle/spconv_cases.py -- row counts on the 64-row tiles, the 256-row weight-gradient slabs and their 32-row steps, the
row bounds met with equality, extents of 1 and 2, batches with an empty frame, duplicate points.

(a) Eval mode in the affine regime (small gamma, large beta: every pre-activation is asserted to be more than ten times
    the comparator's bound, so no fp32 rounding flips a ReLU): the four volumes, the code gradient and all 51 parameter
    gradients within kappa 2^-24 t of float64, t from the absolute-value twin.
(b) Train mode: volumes element-wise, running statistics, gradients tensor by tensor against the float64 emulation.
(c) Cotangents on some volumes only: the others reach the kernel as NULL.
(d) Every output element written, nothing written past the workspace.
(e) Replays: the forward is bit-identical, two backwards agree within the gate."""
import ctypes

import pytest
import torch

from neuralbody_b200 import capi
from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet, _Encode
from oracle import spconv_cases as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = S.all_cases()
CHANNELS = (32, 64, 128, 128)


def _nets(seed, gamma, beta):
    """(float32 DenseSparseConvNet on the GPU, CudaSparseConvNet with the same values), random running statistics."""
    torch.manual_seed(seed)
    net = DenseSparseConvNet()
    with torch.no_grad():
        for _, bn in S.layers(net):
            bn.weight.uniform_(*gamma)
            bn.bias.uniform_(*beta)
            bn.running_mean.uniform_(-0.5, 0.5)
            bn.running_var.uniform_(0.5, 2.0)
    ours = CudaSparseConvNet()
    ours.load_state_dict(net.state_dict())
    return net.to(DEV), ours.to(DEV)


def _affine(seed):
    return _nets(seed, (0.005, 0.015), (2.5, 3.5))


def _inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    code = torch.randn(c["n_vert"], 16, generator=g).to(DEV)
    cots = [torch.randn((c["B"], ch) + s, generator=g).to(DEV)
            for ch, s in zip(CHANNELS, S.level_shapes(c["out_sh"])[1:])]
    return code, cots


def _ours(net, c, code, cots):
    """CudaSparseConvNet's volumes and gradients for the cotangents `cots` (None: that volume is not differentiated)."""
    code = code.clone().requires_grad_(True)
    vols = net.encode(code, c["coord"].to(DEV), c["out_sh"], c["B"])
    pairs = [(v, t) for v, t in zip(vols, cots) if t is not None]
    torch.autograd.backward([v for v, _ in pairs], [t for _, t in pairs])
    out = {"net%d" % (l + 1): v.detach() for l, v in enumerate(vols)}
    out["code"] = code.grad
    named = dict(net.named_parameters())
    out.update({k: named[k].grad for k in S.param_names()})
    return out


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _check_counts(net, c):
    assert net.last_row_counts.cpu().tolist() == c["counts"], (c["name"], net.last_row_counts.tolist(), c["counts"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_eval_affine_regime_matches_float64_element_by_element(built_lib, name):
    c = CASES[name]
    net, ours = _affine(1)
    ours.eval()
    code, cots = _inputs(c, 2)
    want, t, margin = S.reference_and_twin(net.eval(), code, c["coord"].to(DEV), c["out_sh"], c["B"], cots)
    assert margin > 10, "%s: a pre-activation is within %.1f x the gate of its ReLU" % (name, margin)
    got = _ours(ours, c, code, cots)
    _check_counts(ours, c)
    ratios = S.compare_all(got, want, t, c["counts"], name)
    worst = max(ratios, key=ratios.get)
    print("\n%s: margin %.0f, worst ratio %.2e (%s)" % (name, margin, ratios[worst], worst))
    # the element-wise gate of a weight several layers from every volume is loose (its twin cotangent went through |W|
    # where the real one cancels): those gradients are held to a relative L2 of 1e-4 as well
    for k in ["code"] + S.param_names():
        assert torch.isfinite(got[k]).all() and _rel_l2(got[k], want[k]) <= 1e-4, (name, k, _rel_l2(got[k], want[k]))


def _train_margin(net, c, code):
    """min over active rows and channels of every layer of the float64 train-mode pre-activation."""
    emu = S.emulation(net).train()
    emu.pre = []
    with torch.no_grad():
        emu.encode(code.double(), c["coord"].to(DEV), c["out_sh"], c["B"])
    return min(float(p[(m > 0).expand_as(p)].min()) for p, m in emu.pre)


@pytest.mark.parametrize("name", sorted(CASES))
def test_train_mode_matches_float64(built_lib, name):
    c = CASES[name]
    if min(c["counts"]) < 3:
        # one row: BatchNorm1d refuses it in training.  Two rows: BatchNorm maps them to +-gamma d / sqrt(d^2 + eps) + beta,
        # so every gradient through it is a cancellation residue of relative size eps / (d^2 + eps), rounding noise in fp32
        pytest.skip("a level with fewer than three active rows: train-mode BatchNorm has no fp32-comparable reference there")
    net, ours = _nets(3, (0.05, 0.1), (2.5, 3.5))
    code, cots = _inputs(c, 4)
    # the ReLUs stay open by a margin far above any fp32 difference, so the float64 and fp32 runs take the same branches
    assert _train_margin(net, c, code) > 0.05
    ref = S.emulation(net).train()
    want = S.run(ref, code.double(), c["coord"].to(DEV), c["out_sh"], c["B"], cots)
    f32 = S.emulation(net, torch.float32).train()
    saved = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        emu32 = S.run(f32, code, c["coord"].to(DEV), c["out_sh"], c["B"], cots)
    finally:
        torch.backends.cudnn.allow_tf32 = saved
    got = _ours(ours.train(), c, code, cots)
    _check_counts(ours, c)
    for l in range(4):
        k = "net%d" % (l + 1)
        gamma = S.layers(net)[S.OUT_LAYERS[l]][1].weight.detach().double().view(1, -1, 1, 1, 1)
        err = (got[k].double() - want[k]).abs()
        tol = 1e-4 * (want[k].abs() + gamma)
        assert bool((err <= tol).all()), "%s %s: worst |error| / tol %.2f" % (name, k, float((err / tol).max()))
    sd_ref, sd_ours = ref.state_dict(), ours.state_dict()
    for k in sd_ref:
        if "running" in k:
            assert _rel_l2(sd_ours[k], sd_ref[k]) <= 1e-5, (name, k, _rel_l2(sd_ours[k], sd_ref[k]))
        if "num_batches_tracked" in k:
            assert int(sd_ours[k]) == int(sd_ref[k]) == 1, (name, k)
    # Where a level's rows are isolated, a SubM layer acts row by row and the next BatchNorm removes any per-channel constant
    # (d beta of the layer before is exactly 0, and weights several such layers deep get the same cancellation): the float64
    # value there is a residue that fp32 rounding swamps -- the fp32 emulation itself is > 1e-2 off.  Such a tensor is held to
    # the emulation's noise level, an order of magnitude in the summation order; every other one to max(1e-4, 2 x its error).
    resolved = 0
    for k in ["code"] + S.param_names():
        e32, err = _rel_l2(emu32[k], want[k]), _rel_l2(got[k], want[k])
        assert torch.isfinite(got[k]).all(), (name, k)
        if e32 <= 1e-2:
            resolved += 1
            assert err <= max(1e-4, 2 * e32), (name, k, err, e32)
        else:
            assert err <= 10 * e32, (name, k, err, e32)
    assert resolved >= 17, (name, resolved)


@pytest.mark.parametrize("levels", ((0,), (3,), (1, 2)))
@pytest.mark.parametrize("name", ("odd40", "batch5", "tile257"))
def test_volumes_without_a_cotangent_reach_the_kernel_as_null(built_lib, monkeypatch, name, levels):
    c = CASES[name]
    net, ours = _affine(5)
    ours.eval()
    code, cots = _inputs(c, 6)
    cots = [t if l in levels else None for l, t in enumerate(cots)]
    seen = []
    backward = _Encode.backward

    def spy(ctx, *d_vols):
        seen.append([d is not None for d in d_vols])
        return backward(ctx, *d_vols)
    monkeypatch.setattr(_Encode, "backward", staticmethod(spy))
    got = _ours(ours, c, code, cots)
    assert seen == [[l in levels for l in range(4)]], seen
    zero = [torch.zeros_like(v) if t is None else t for v, t in zip(got.values(), cots)]
    want, t, margin = S.reference_and_twin(net.eval(), code, c["coord"].to(DEV), c["out_sh"], c["B"], zero)
    assert margin > 10, margin
    ratios = S.compare_all(got, want, t, c["counts"], "%s %s" % (name, levels))
    print("\n%s cotangents on %s: worst ratio %.2e" % (name, levels, max(ratios.values())))


def _raw_args(ours, c, code):
    """nb_spconv_args for ours (eval mode) as _Encode builds them, plus the tensors behind its pointers."""
    a = capi.nb_spconv_args()
    a.batch, a.n_points, a.n_vert = c["B"], c["coord"].shape[0], c["n_vert"]
    for i in range(3):
        a.out_sh[i] = c["out_sh"][i]
    coord = c["coord"].to(DEV).contiguous()
    a.coord, a.code = coord.data_ptr(), code.data_ptr()
    pairs = ours.convs_and_batchnorms()
    for j, (conv, bn) in enumerate(pairs):
        a.weight[j], a.bn_weight[j], a.bn_bias[j] = conv.weight.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr()
        a.running_mean[j], a.running_var[j] = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
        a.num_batches_tracked[j] = bn.num_batches_tracked.data_ptr()
    a.training, a.momentum, a.eps = 0, pairs[0][1].momentum, pairs[0][1].eps
    return a, coord


def _poison(t):
    """0xFF bytes: NaN as float, -1 as int."""
    t.view(torch.uint8).fill_(0xFF)
    return t


@pytest.mark.parametrize("name", ("tile257", "filled_b2", "duplicates", "extent111", "odd40"))
def test_every_output_is_written_and_nothing_past_the_workspace(built_lib, name):
    c = CASES[name]
    net, ours = _affine(7)
    code, cots = _inputs(c, 8)
    lib = capi.load()
    a, coord = _raw_args(ours, c, code)
    need = lib.nb_spconv_workspace_bytes(a.batch, a.n_points, a.out_sh)
    tail = 1 << 20
    ws = _poison(torch.empty(need + tail, dtype=torch.uint8, device=DEV))
    pattern = (torch.arange(tail, device=DEV) * 7 % 251).to(torch.uint8)
    ws[need:] = pattern
    a.workspace, a.workspace_bytes = ws.data_ptr(), need
    vols = [_poison(torch.empty((c["B"], ch) + s, device=DEV)) for ch, s in zip(CHANNELS, S.level_shapes(c["out_sh"])[1:])]
    for l, v in enumerate(vols):
        a.volumes[l] = v.data_ptr()
    counts = _poison(torch.empty(5, dtype=torch.int32, device=DEV))
    a.row_counts = counts.data_ptr()
    g = capi.nb_spconv_grads()
    for l, t in enumerate(cots):
        g.d_volumes[l] = t.data_ptr()
    d_code = _poison(torch.empty_like(code))
    g.d_code = d_code.data_ptr()
    params = [p for conv, bn in ours.convs_and_batchnorms() for p in (conv.weight, bn.weight, bn.bias)]
    grads = [_poison(torch.empty_like(p)) for p in params]
    for j in range(17):
        g.d_weight[j], g.d_bn_weight[j], g.d_bn_bias[j] = (grads[3 * j + i].data_ptr() for i in range(3))
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    capi.check(lib.nb_spconv_fwd(ctypes.byref(a), stream), "nb_spconv_fwd")
    capi.check(lib.nb_spconv_bwd(ctypes.byref(a), ctypes.byref(g), stream), "nb_spconv_bwd")
    torch.cuda.synchronize()
    assert counts.cpu().tolist() == c["counts"]
    for v, m in zip(vols, S.masks(c["coord"], c["out_sh"], c["B"], DEV)[1:]):
        assert torch.isfinite(v).all()
        assert float((v.double() * (1 - m)).abs().max()) == 0.0
        assert bool(((v != 0).any(1, keepdim=True) == (m > 0)).all())      # beta = 3: every active row is non-zero
    for t in [d_code] + grads:
        assert torch.isfinite(t).all()
    assert torch.equal(ws[need:], pattern), "the kernels wrote past the workspace"


@pytest.mark.parametrize("name", ("tile289", "batch5"))
def test_replays(built_lib, name):
    """An eval-mode forward has no atomics: repeated, it is bit-identical.  The backward reads only what the forward
    saved: run twice on one graph, it agrees with itself within the gate."""
    c = CASES[name]
    net, ours = _affine(9)
    ours.eval()
    code, cots = _inputs(c, 10)
    coord = c["coord"].to(DEV)
    with torch.no_grad():
        first = ours.encode(code, coord, c["out_sh"], c["B"])
        second = ours.encode(code, coord, c["out_sh"], c["B"])
    assert all(torch.equal(x, y) for x, y in zip(first, second))
    code_ = code.clone().requires_grad_(True)
    vols = ours.encode(code_, coord, c["out_sh"], c["B"])
    runs = []
    for _ in range(2):
        code_.grad = None
        ours.zero_grad(set_to_none=True)
        torch.autograd.backward(vols, cots, retain_graph=True)
        named = dict(ours.named_parameters())
        runs.append(dict([("code", code_.grad.clone())] + [(k, named[k].grad.clone()) for k in S.param_names()]))
    _, t, _ = S.reference_and_twin(net.eval(), code, coord, c["out_sh"], c["B"], cots)
    for k in runs[0]:
        S.check_elementwise(runs[1][k], runs[0][k], t[k], S.kappa(k, c["counts"]), "%s replay %s" % (name, k))
