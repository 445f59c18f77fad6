"""Edge cases, an absolute-value twin and an element-wise comparator for the sparse CUDA encoder (csrc/nb_spconv.cu).

Cases.  Each builder returns a dict: `coord` int32 (n, 4) = (frame, z, y, x), `out_sh`, `B`, `n_vert` (point i takes
code[i % n_vert]), `counts` = the active sites of the input grid and the four strided levels (what nb_spconv_fwd writes to
row_counts) from the float64 masks, and `promise` = {level: count} that the construction aims at.  The constructions:
a point at an even coordinate feeds one stride-2 output per axis, so points on a lattice of step 2^s keep their count
for s levels; a point at an odd coordinate feeds two per axis, so isolated odd points give level 1 exactly 8 x n_points
rows (nb_spconv's row bound with equality); a filled grid has every site of every level active.

Twin.  `abs_twin` is DenseSparseConvNet in float64 with |W|, |code|, each eval-mode BatchNorm replaced by
(x + |mean|) |gamma istd| + |beta| and no ReLU.  Its outputs, and its gradients for the cotangent |cot|, are for every
element the sum t of the magnitudes of the product terms the element is made of (in eval mode, with every ReLU passing,
the encode is a polynomial in code, the weights, gamma, beta and the cotangent; the twin evaluates each of its monomials
in magnitude).

Comparator.  `check_elementwise(got, ref64, t, kappa)` asserts |got - ref64| <= kappa 2^-24 t element by element.  Each
fp32 operation rounds with a relative error <= u = 2^-24, so a term that passes through m roundings is perturbed by a
factor within (1 +- u)^m, and the computed element is within gamma_m t of the exact one, gamma_m = m u / (1 - m u)
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 3.1, 3.3), whatever the summation order.  kappa is
that m, counted along the longest chain: a convolution adds at most 27 Cin products into one output (27 Cout for its
data gradient), BatchNorm rounds a term at most 4 times (mean subtraction, istd, gamma, beta; istd itself is rounded to
float once), a weight gradient adds up to one product per row of its level, the code gradient one per row sharing a
vertex.  For the whole network the forward chain is sum_j (27 Cin_j + 4) = 35060; `kappa()` gives it per output tensor.
m u <= 4.5e-3 here, so 1 / (1 - m u) is folded into kappa by rounding up.  The float64 reference's own error is ~1e-16
relative and is not counted."""
import numpy as np
import torch
import torch.nn.functional as F

from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet, _masked_bn_relu

U = 2.0 ** -24
BLOCKS = ("conv0", "down0", "conv1", "down1", "conv2", "down2", "conv3", "down3", "conv4")
CIN = (16, 16, 16, 32, 32, 32, 64, 64, 64, 64, 128, 128, 128, 128, 128, 128, 128)
COUT = (16, 16, 32, 32, 32, 64, 64, 64, 64, 128, 128, 128, 128, 128, 128, 128, 128)
STRIDE = (1, 1, 2, 1, 1, 2, 1, 1, 1, 2, 1, 1, 1, 2, 1, 1, 1)
OUT_LAYERS = (4, 8, 12, 16)                        # net1..net4 are the outputs of these layers
LEVEL_OUT = tuple(int(np.cumsum([s == 2 for s in STRIDE])[j]) for j in range(17))    # grid level of layer j's rows
BN_ROUNDINGS = 4


def layers(net):
    """The 17 (conv, BatchNorm1d) pairs of a DenseSparseConvNet in the network's order."""
    out = []
    for name in BLOCKS:
        blk = getattr(net, name)
        out += [(blk[i], blk[i + 1]) for i in range(0, len(blk), 3)]
    return out


def param_names():
    """state-dict names of the 17 conv weights, the 17 BatchNorm weights and the 17 BatchNorm biases, in the kernel's
    order (CudaSparseConvNet's params)."""
    convs = ["%s.%d" % (name, 3 * i) for name, n in zip(BLOCKS, (2, 1, 2, 1, 3, 1, 3, 1, 3)) for i in range(n)]
    bns = ["%s.%d" % (c.split(".")[0], int(c.split(".")[1]) + 1) for c in convs]
    return [c + ".weight" for c in convs] + [b + ".weight" for b in bns] + [b + ".bias" for b in bns]


# ---------------------------------------------------------------------------------------------------------------- kappa

def _fwd_chain(j):
    """Roundings on the longest chain into layer j's input rows."""
    return sum(27 * CIN[i] + BN_ROUNDINGS for i in range(j))


def _bwd_chain(j):
    """Roundings on the longest chain of the cotangent of layer j's convolution output: the data gradients of the later
    layers, every BatchNorm backward on the way and the volume cotangents added in."""
    return sum(27 * COUT[i] + BN_ROUNDINGS for i in range(j + 1, 17)) + BN_ROUNDINGS + len(OUT_LAYERS)


def kappa(name, counts):
    """kappa of one compared tensor: 'net1'..'net4', 'code' or a parameter name; counts = the case's row counts."""
    if name.startswith("net"):
        m = _fwd_chain(OUT_LAYERS[int(name[3:]) - 1] + 1)
    elif name == "code":
        m = _bwd_chain(0) + 27 * COUT[0] + counts[0]
    else:
        i = param_names().index(name)
        j = i % 17
        if i >= 17:                                # BatchNorm gamma / beta: sums in float64, rounded to float once
            m = _fwd_chain(j + 1) + _bwd_chain(j) + 1
        else:
            m = _fwd_chain(j) + _bwd_chain(j) + counts[LEVEL_OUT[j]]
    return float(np.ceil(m * 1.005))


KAPPA_FWD = _fwd_chain(17)


def check_elementwise(got, ref64, twin, kappa_, label=""):
    """Assert |got - ref64| <= kappa_ 2^-24 twin for every element (NaN fails); return the worst |got - ref64| / bound."""
    got, ref, t = got.detach().double(), ref64.detach().double(), twin.detach().double()
    assert got.shape == ref.shape == t.shape, (label, got.shape, ref.shape, t.shape)
    err = (got - ref).abs()
    bound = kappa_ * U * t
    ok = err <= bound
    if not bool(ok.all()):
        i = int((~ok).flatten().nonzero()[0])
        idx = np.unravel_index(i, tuple(got.shape))
        raise AssertionError("%s: %d elements outside kappa %.0f u t; first at %s: got %.9g, float64 %.9g, bound %.3g" % (
            label, int((~ok).sum()), kappa_, idx, float(got.flatten()[i]), float(ref.flatten()[i]),
            float(bound.flatten()[i])))
    pos = bound > 0
    return float((err[pos] / bound[pos]).max()) if bool(pos.any()) else 0.0


# ------------------------------------------------------------------------------------------------------------ emulation

def _eval_bn_relu(bn, x, mask, pre=None):
    C = x.shape[1]
    y = (x - bn.running_mean.view(1, C, 1, 1, 1)) * torch.rsqrt(bn.running_var.view(1, C, 1, 1, 1) + bn.eps)
    y = y * bn.weight.view(1, C, 1, 1, 1) + bn.bias.view(1, C, 1, 1, 1)
    if pre is not None:
        pre.append((y.detach(), mask))
    return F.relu(y) * mask


def _train_bn_relu(bn, x, mask, pre=None):
    if pre is not None:
        with torch.no_grad():
            C, n = x.shape[1], mask.sum().clamp_min(1.0)
            mean = x.sum(dim=(0, 2, 3, 4)) / n
            var = (((x - mean.view(1, C, 1, 1, 1)) * mask) ** 2).sum(dim=(0, 2, 3, 4)) / n
            y = (x - mean.view(1, C, 1, 1, 1)) * torch.rsqrt(var.view(1, C, 1, 1, 1) + bn.eps)
            pre.append((y * bn.weight.view(1, C, 1, 1, 1) + bn.bias.view(1, C, 1, 1, 1), mask))
    return _masked_bn_relu(bn, x, mask)


def _twin_bn(bn, x, mask, pre=None):
    C = x.shape[1]
    istd = torch.rsqrt(bn.running_var.view(1, C, 1, 1, 1) + bn.eps)
    y = (x + bn.running_mean.abs().view(1, C, 1, 1, 1)) * (bn.weight.view(1, C, 1, 1, 1) * istd).abs()
    y = y + bn.bias.abs().view(1, C, 1, 1, 1)
    if pre is not None:
        pre.append((y.detach(), mask))
    return y * mask


class Emulation(DenseSparseConvNet):
    """DenseSparseConvNet's encode, layer by layer: `conv_hook(j, x_in, x_out, conv, mask_in, mask_out) -> x_out` runs after
    each convolution, and `pre` (a list) receives every layer's (pre-activation, active mask) when set.  `twin` selects the
    absolute-value BatchNorm; otherwise BatchNorm + ReLU follow the module's train / eval mode."""

    def __init__(self):
        super().__init__()
        self.conv_hook, self.pre, self.twin = None, None, False

    def forward(self, x, mask):
        outs = []
        for j, (conv, bn) in enumerate(layers(self)):
            x_in, m_in = x, mask
            x, mask = conv(x, mask)
            if self.conv_hook is not None:
                x = self.conv_hook(j, x_in, x, conv, m_in, mask)
            bn_act = _twin_bn if self.twin else (_train_bn_relu if bn.training else _eval_bn_relu)
            x = bn_act(bn, x, mask, self.pre)
            if j in OUT_LAYERS:
                outs.append(x)
        return outs


def emulation(net, dtype=torch.float64):
    """An Emulation holding net's parameters and statistics in `dtype`, in net's train / eval mode."""
    emu = Emulation()
    emu.load_state_dict(net.state_dict())
    return emu.to(device=next(net.parameters()).device, dtype=dtype).train(net.training)


def abs_twin(net):
    """The absolute-value twin of net (eval mode, float64)."""
    tw = emulation(net).eval()
    tw.twin = True
    with torch.no_grad():
        for conv, bn in layers(tw):
            conv.weight.abs_()
            bn.weight.abs_()
            bn.bias.abs_()
    return tw


def run(emu, code, coord, out_sh, B, cots):
    """Volumes and gradients of emu: {'net1'..'net4', 'code', parameter names} for the cotangents `cots` (None = 0)."""
    code = code.detach().clone().requires_grad_(True)
    for p in emu.parameters():
        p.grad = None
    vols = emu.encode(code, coord, out_sh, B)
    pairs = [(v, c.to(v.dtype)) for v, c in zip(vols, cots) if c is not None]
    torch.autograd.backward([v for v, _ in pairs], [c for _, c in pairs])
    out = {"net%d" % (l + 1): v.detach() for l, v in enumerate(vols)}
    out["code"] = code.grad
    named = dict(emu.named_parameters())
    for k in param_names():
        g = named[k].grad
        out[k] = torch.zeros_like(named[k]) if g is None else g
    return out


def reference_and_twin(net, code, coord, out_sh, B, cots):
    """(float64 emulation results, twin results, margin) for an eval-mode net: margin = min over the active rows and
    channels of every layer of the float64 pre-activation / (KAPPA_FWD u t); > 10 keeps every ReLU open under fp32."""
    ref = emulation(net).eval()
    ref.pre = []
    want = run(ref, code.double(), coord, out_sh, B, cots)
    tw = abs_twin(net)
    tw.pre = []
    t = run(tw, code.double().abs(), coord, out_sh, B, [None if c is None else c.abs() for c in cots])
    return want, t, affine_margin(ref.pre, tw.pre)


def affine_margin(pre, twin_pre):
    worst = float("inf")
    for (p, m), (t, _) in zip(pre, twin_pre):
        act = (m > 0).expand_as(p)
        worst = min(worst, float((p[act] / (KAPPA_FWD * U * t[act])).min()))
    return worst


def compare_all(got, want, twin, counts, label=""):
    """check_elementwise on every tensor of `want`; returns {name: worst ratio}."""
    return {k: check_elementwise(got[k], want[k], twin[k], kappa(k, counts), "%s %s" % (label, k)) for k in want}


# ---------------------------------------------------------------------------------------------------------------- masks

def level_shapes(out_sh):
    shapes, cur = [tuple(int(v) for v in out_sh)], [int(v) for v in out_sh]
    for _ in range(4):
        cur = [(v - 1) // 2 + 1 for v in cur]
        shapes.append(tuple(cur))
    return shapes


def masks(coord, out_sh, B, device="cpu"):
    """The active set of the input grid and of every level, (B, 1, D, H, W) float64, by the emulation's rules."""
    D, H, W = (int(v) for v in out_sh)
    c = coord.long().to(device)
    m = torch.zeros((B, 1, D, H, W), dtype=torch.float64, device=device)
    m[c[:, 0], 0, c[:, 1], c[:, 2], c[:, 3]] = 1.0
    out = [m]
    for _ in range(4):
        m = F.max_pool3d(m, 3, stride=2, padding=1)
        out.append(m)
    return out


def row_bounds(B, n_points, out_sh):
    """nb_spconv's static row bounds: level 0 <= n_points, level l+1 <= min(8 x level l, sites)."""
    caps = []
    for l, s in enumerate(level_shapes(out_sh)):
        sites = B * s[0] * s[1] * s[2]
        caps.append(min(n_points if l == 0 else 8 * caps[-1], sites))
    return caps


# ---------------------------------------------------------------------------------------------------------------- cases

def _case(name, coord, out_sh, B, n_vert, promise):
    coord = torch.as_tensor(np.asarray(coord), dtype=torch.int32).reshape(-1, 4)
    counts = [int(m.sum()) for m in masks(coord, out_sh, B)]
    return {"name": name, "coord": coord, "out_sh": [int(v) for v in out_sh], "B": int(B), "n_vert": int(n_vert),
            "counts": counts, "promise": dict(promise)}


def _lattice_points(n, step, dims, offset=0):
    """The first n points, in site order, of a lattice dims[0] x dims[1] x dims[2] of the given step."""
    pts = [(offset + step * a, offset + step * b, offset + step * c)
           for a in range(dims[0]) for b in range(dims[1]) for c in range(dims[2])]
    assert len(pts) >= n
    return pts[:n]


def lattice(name, n, step, dims, levels, B=1, n_vert=None):
    """n points on a lattice of step 2^s (s >= levels - 1), frame B - 1: the first `levels` levels hold n rows each."""
    pts = _lattice_points(n, step, dims)
    out_sh = [step * (d - 1) + 1 for d in dims]
    coord = [(B - 1,) + p for p in pts]
    return _case(name, coord, out_sh, B, n_vert or n, {l: n for l in range(levels)})


def isolated_odd(name, n, dims):
    """n points at odd coordinates 4 i + 1: level 1 has exactly 8 n rows, the row bound's 8 x n_points."""
    pts = _lattice_points(n, 4, dims, offset=1)
    out_sh = [4 * d + 1 for d in dims]            # room for both outputs of the last point, and more level-1 sites
    return _case(name, [(0,) + p for p in pts], out_sh, 1, n, {0: n, 1: 8 * n})


def filled(name, out_sh, B):
    """Every site of every frame active: each level's count is its number of sites, and the last site is active."""
    g = np.stack(np.meshgrid(np.arange(B), *[np.arange(s) for s in out_sh], indexing="ij"), -1).reshape(-1, 4)
    return _case(name, g, out_sh, B, len(g), {l: B * int(np.prod(s)) for l, s in enumerate(level_shapes(out_sh))})


def random_points(name, out_sh, B, n, seed, frames=None, last_site=True, n_vert=None):
    """n random points (with repeats) in the frames `frames` (default all), plus the grid's last site when last_site."""
    g = np.random.default_rng(seed)
    frames = list(range(B)) if frames is None else frames
    pts = np.stack([g.choice(frames, n)] + [g.integers(0, s, n) for s in out_sh], 1)
    if last_site:
        pts = np.concatenate([pts, [[B - 1] + [s - 1 for s in out_sh]]])
    return _case(name, pts, out_sh, B, n_vert or len(pts), {})


def boxes(name, out_sh, B, frame_boxes, seed, n_vert=None):
    """Frames filled on boxes {frame: (lo, hi)} (inclusive), the points in a random order across the frames."""
    pts = []
    for b, (lo, hi) in frame_boxes.items():
        g = np.stack(np.meshgrid(*[np.arange(l, h + 1) for l, h in zip(lo, hi)], indexing="ij"), -1).reshape(-1, 3)
        pts.append(np.concatenate([np.full((len(g), 1), b), g], 1))
    pts = np.concatenate(pts)
    pts = pts[np.random.default_rng(seed).permutation(len(pts))]
    n0 = sum(int(np.prod([h - l + 1 for l, h in zip(lo, hi)])) for lo, hi in frame_boxes.values())
    return _case(name, pts, out_sh, B, n_vert or len(pts), {0: n0})


def duplicates(name, seed):
    """Two frames whose points share sites 1 to 6 times each, interleaved across the frames, the code indexed modulo a
    smaller n_vert: the highest point index wins a site, and it is rarely the frame's last point."""
    g = np.random.default_rng(seed)
    out_sh = (17, 9, 6)
    sites = []
    for b in range(2):
        flat = g.choice(int(np.prod(out_sh)), 45, replace=False)
        sites += [(b,) + tuple(int(v) for v in np.unravel_index(f, out_sh)) for f in flat]
    pts = [s for s in sites for _ in range(int(g.integers(1, 7)))]
    pts = np.asarray(pts)[g.permutation(len(pts))]
    return _case(name, pts, out_sh, 2, 37, {0: len(sites)})


def tile_edge(n):
    """Level 0 with n rows: the first n sites of a filled box (full 27-neighbourhoods inside), the rest of the grid empty."""
    dims = {1: (1, 1, 1), 63: (3, 3, 7), 64: (4, 4, 4), 65: (5, 4, 4), 255: (15, 17, 1), 256: (4, 8, 8), 257: (5, 8, 8),
            288: (6, 6, 8), 289: (17, 17, 1)}[n]
    pts = _lattice_points(n, 1, dims, offset=1)
    out_sh = [d + 2 for d in dims]
    return _case("tile%d" % n, [(0,) + p for p in pts], out_sh, 1, n, {0: n})


def all_cases():
    """Every case, by name."""
    cases = [tile_edge(n) for n in (1, 63, 64, 65, 255, 256, 257, 288, 289)]
    cases += [
        lattice("lattice4_63", 63, 4, (7, 9, 1), 3),              # levels 0-2: 63 rows
        lattice("lattice16_64", 64, 16, (4, 4, 4), 5),            # every level: 64 rows
        lattice("lattice8_65", 65, 8, (5, 13, 1), 4, B=2),        # levels 0-3: 65 rows, all in frame 1
        isolated_odd("odd40", 40, (4, 5, 2)),                     # level 1: 320 = 8 x n_points rows
        filled("filled_b2", (17, 10, 9), 2),                      # every level full, the min(., sites) bound binds
        filled("extent111", (1, 1, 1), 1),
        filled("extent152", (1, 5, 2), 1),
        random_points("extent237", (2, 3, 7), 1, 20, 1),
        random_points("extent33_1_17", (33, 1, 17), 1, 200, 2),
        random_points("extent41_39_43", (41, 39, 43), 1, 700, 3),
        boxes("batch3", (20, 9, 14), 3, {0: ((0, 0, 0), (11, 4, 6)), 2: ((3, 2, 5), (7, 8, 13))}, 4),
        boxes("batch5", (10, 12, 11), 5, {0: ((0, 0, 0), (3, 3, 3)), 1: ((2, 5, 1), (9, 11, 4)),
                                          3: ((0, 0, 9), (2, 2, 10)), 4: ((4, 4, 4), (9, 6, 10))}, 5, n_vert=61),
        duplicates("duplicates", 6),
    ]
    return {c["name"]: c for c in cases}
