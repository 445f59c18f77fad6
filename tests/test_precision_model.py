"""CPU: the NUMERICAL DESIGN of the tensor-core decoder, checked against the reference's golden vectors without a GPU.

The CUDA decoder (neuralbody_b200/csrc/nb_render_tc_list.cu) cannot run here, but every rounding it applies can be restated:
operands of layers 0-2 (the density path, latent_xyzc.py:99-104) travel as fp16 (hi, lo) pairs -- hi = the value truncated to
fp16, lo = fp16(value - hi) -- and the tensor cores accumulate A_hi W_hi + A_lo W_hi + A_hi W_lo in fp32; h2 enters the folded
colour layer (latent_xyzc.py:106-121, folded as nb_layout.h describes) as ONE fp16 rounded to nearest; alpha_fc and rgb_fc are
fp32 dot products.  This module emulates exactly those roundings around the oracle's own feature gather and compositing, on the
full-size `full_313` golden case (the scene on which the 1-pass mode misses the gate), and pins the two facts the kernel's
precision scheme rests on (the emulation itself lives in oracle/tc_decoder_model.py, which tests/test_decoder_rows_gpu.py
also holds the kernel to row by row):

  * the 3-pass scheme with a 1-pass colour layer stays well inside the north star's 1e-3 gate on every map;
  * one fp16 rounding per density-path operand (the 1-pass `tc_fp16` mode) does NOT: its depth error is several times larger,
    which is why the default mode pays 2.7x the algorithmic tensor FLOPs.

Test infrastructure only (it imports oracle/); nothing here is product code.
"""
import numpy as np
import torch

from conftest import golden_case
from oracle import neuralbody_oracle as O
from oracle import tc_decoder_model as M


def _decode(scene, wpts, viewdir, density_passes):
    """(P,3) world points / view directions of ONE frame -> raw (P,4) with the decoder's roundings, on the oracle's gather."""
    sp = O.prepare_sp_input(scene)
    ppts = O.pts_to_can_pts(wpts[None], sp["R"], sp["Th"])
    grid = O.get_grid_coords(ppts, sp["bounds"], sp["out_sh"], scene["voxel_size"])
    f = O.interpolate_features(grid, scene["volumes"])[0].t().contiguous()            # (P,352) fp32, as the producers gather it
    pe = torch.cat([O.positional_embed(viewdir, 4), O.positional_embed(wpts, 10)], -1)  # order of latent_xyzc.py:117-119
    return M.decode_rows(scene["weights"], int(scene["latent_index"].reshape(-1)[0]), f, pe=pe, passes=density_passes)


def _render(scene, n_samples, density_passes):
    assert scene["ray_o"].shape[0] == 1
    wpts, z_vals = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], n_samples)
    viewdir = scene["ray_d"] / torch.norm(scene["ray_d"], dim=2, keepdim=True)
    n = wpts.shape[1]
    vd = viewdir[:, :, None].expand(1, n, n_samples, 3).reshape(-1, 3)
    raw = _decode(scene, wpts.reshape(-1, 3), vd, density_passes).reshape(n, n_samples, 4)
    rgb, disp, acc, weights, depth = O.raw2outputs(raw, z_vals.view(-1, n_samples), scene["ray_d"].reshape(-1, 3))
    return {"rgb_map": rgb.numpy(), "acc_map": acc.numpy(), "depth_map": depth.numpy()}


def _max_abs(out, gold):
    return {k: float(np.abs(out[k] - gold[k].reshape(out[k].shape)).max()) for k in out}


def test_split_is_exact_and_13_bits_survive():
    """hi + lo reproduces an fp32 value to ~2^-22 relative (hi keeps 11 bits by truncation, lo the next 11)."""
    g = torch.Generator().manual_seed(5)
    x = (torch.rand(4096, generator=g) * 8 - 4)
    hi, lo = M.split_act(x)
    assert torch.equal(hi, hi.to(torch.float16).to(torch.float32))                     # hi is representable in fp16
    assert float((hi.abs() <= x.abs()).float().min()) == 1.0                           # truncation, not rounding
    rel = ((hi + lo - x).abs() / x.abs().clamp_min(1e-3)).max()
    assert float(rel) < 2.0 ** -20


def test_three_pass_scheme_meets_the_gate_and_one_pass_does_not():
    scene, rkw, gold = golden_case("full_313")
    e3 = _max_abs(_render(scene, rkw["n_samples"], 3), gold)
    e1 = _max_abs(_render(scene, rkw["n_samples"], 1), gold)
    print("precision model on full_313 (max abs vs the reference): 3-pass %s | 1-pass %s" % (e3, e1))
    # the north star's gate is 1e-3 on every map; the GPU tests hold the kernel to it (tests/test_render_gpu.py)
    assert e3["rgb_map"] < 5e-4 and e3["depth_map"] < 2e-4 and e3["acc_map"] < 1e-4, e3
    # one fp16 rounding per density-path operand moves the depth by several gate widths' worth more
    assert e1["depth_map"] > 5 * e3["depth_map"] and e1["depth_map"] > 5e-4, (e1, e3)
