"""CPU: the masked demo renderers with coarse + fine sampling (f-1 x f-4, oracle/masked_hier_case.py).  The oracle's
restatement against the golden vectors made by composing the unmodified reference's own masked renderer, sample_pdf and
sort-merge; and the properties that make the cases worth testing."""
import numpy as np
import pytest

from conftest import load_golden
from oracle import masked_hier_case as MH, neuralbody_oracle as O, synth

KEYS = ("rgb_map", "disp_map", "acc_map", "weights", "depth_map", "rgb0", "disp0", "acc0", "z_std", "z_vals", "weights0")


def _case(name):
    scene, rkw = MH.build_case(name)
    gold = load_golden(name)
    assert synth.scene_checksum(scene) == gold["input_sha256"], "rebuilt inputs differ from the golden generator's"
    assert MH.mask_checksum(scene, rkw["masks"]) == bytes(gold["mask_sha256"]).decode()
    return scene, rkw, gold


@pytest.mark.parametrize("name", list(MH.CASES))
def test_masked_hierarchical_oracle_matches_reference_pieces(name):
    scene, rkw, gold = _case(name)
    out = MH.render_hierarchical_masked(scene, rkw["masks"], rkw["n_samples"], rkw["n_importance"])
    for k in KEYS:
        a, b = out[k].numpy(), gold[k]
        assert a.shape == b.shape, k
        # the same torch ops in the same order => bit-identical, NaNs (acc == 0 rays) included
        np.testing.assert_array_equal(np.isnan(a), np.isnan(b))
        np.testing.assert_array_equal(np.nan_to_num(a), np.nan_to_num(b), err_msg=k)
    S, Ni = rkw["n_samples"], rkw["n_importance"]
    assert gold["z_vals"].shape[-1] == S + Ni and (np.diff(gold["z_vals"], axis=-1) >= 0).all()
    assert np.abs(gold["rgb_map"] - gold["rgb0"]).max() > 1e-3      # the fine pass is not a no-op on these scenes


@pytest.mark.parametrize("name", list(MH.CASES))
def test_masks_cut_through_the_body(name):
    """The mask views remove samples the body would otherwise weigh (so the predicate changes the coarse weights the
    sampler reads), and some rays lose every sample in both passes (acc = 0, disp NaN)."""
    scene, rkw, gold = _case(name)
    out = MH.render_hierarchical_masked(scene, rkw["masks"], rkw["n_samples"], rkw["n_importance"])
    ins0, ins = out["inside0"].numpy(), out["inside"].numpy()
    assert 0 < ins0.mean() < 1 and 0 < ins.mean() < 1
    assert (gold["weights0"][~ins0] == 0).all() and (gold["weights"][~ins] == 0).all()
    unmasked = O.render(scene, n_samples=rkw["n_samples"])["weights"].numpy()
    assert (unmasked[~ins0] > 1e-3).any()              # a masked-out sample that the body would have weighed
    dead = ~ins.any(-1) & ~ins0.any(-1)
    assert dead.any() and (gold["acc_map"][dead] == 0).all() and np.isnan(gold["disp_map"][dead]).all()
    assert (gold["acc_map"] > 0.5).any()
