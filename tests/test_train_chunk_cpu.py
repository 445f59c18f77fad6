"""CPU: the full-size training-chunk case (oracle/train_chunk_case.py) is what its GPU test needs it to be.  Every coarse
sample and every importance sample that carries gradient is off the trilinear cell faces and the ReLU kinks (the kinks in
units of the pass's rms pre-activations before its redraws), the conditioning had such samples to move (it is not
vacuous), and the fine depths are a deterministic function of the coarse weights.  The kernel's coarse weights stand in here as the float64 oracle's, rounded to float32."""
import pytest
import torch

from oracle import frames_case as FR
from oracle import train_chunk_case as TC


@pytest.fixture(scope="module")
def scene():
    return TC.full_scene()


@pytest.fixture(scope="module")
def cases(scene):
    return {c: TC.build(c, scene) for c in TC.CHUNK_SEEDS}


def _oracle_coarse_weights(case):
    from oracle import neuralbody_oracle as O
    sc = FR.to_double(case["scene"])
    with torch.no_grad():
        ret = O.get_pixel_value_at(sc["weights"], sc["ray_o"], sc["ray_d"], TC.coarse_depths(case["scene"], case["t_rand"]).double(),
                                   sc["volumes"], O.prepare_sp_input(sc), sc["voxel_size"])
    return ret["weights"].float()


@pytest.mark.parametrize("chunk", sorted(TC.CHUNK_SEEDS))
def test_chunk_is_well_conditioned(cases, chunk):
    case = cases[chunk]
    sc = case["scene"]
    assert tuple(sc["ray_o"].shape) == (1, TC.N_RAYS, 3) and tuple(case["t_rand"].shape) == (1, TC.N_RAYS, TC.N_SAMPLES)
    zc = TC.coarse_depths(sc, case["t_rand"])
    assert not bool(FR.sample_conditions(sc, zc, scale=case["stats"]["coarse"]["scale"])["fragile"].any())
    assert case["stats"]["coarse"]["fragile_first_pass"] > 10, case["stats"]

    w = _oracle_coarse_weights(case)
    u, Z, stats = TC.fine_depths(case, w)
    print(chunk, case["stats"], "fine:", stats)
    assert stats["fragile_first_pass"] > 10, stats
    assert tuple(Z.shape) == (1, TC.N_RAYS, TC.N_SAMPLES + TC.N_IMPORTANCE) and bool((Z[..., 1:] >= Z[..., :-1]).all())
    smp = torch.from_numpy(TC.importance(case, w, u)["z_samples"])[None]
    assert not bool(FR.sample_conditions(sc, smp, scale=stats["scale"])["fragile"].any())
    # the merged depths are the coarse depths and the importance samples, nothing else
    assert torch.equal(torch.sort(torch.cat([zc, smp], -1), -1).values, Z)
    # only the fragile samples' uniforms were redrawn
    changed = int((u != case["u0"]).sum())
    assert 0 < changed < 2 * stats["fragile_first_pass"], (changed, stats)

    # deterministic: the same coarse weights give the same uniforms and depths, bit for bit
    u2, Z2, _ = TC.fine_depths(case, w.clone())
    assert torch.equal(u, u2) and torch.equal(Z.view(torch.int32), Z2.view(torch.int32))


def test_chunks_differ(scene, cases):
    """Chunk B is another set of rays than chunk A (run_c3's chunk), so a Renderer stepping through both sees new lists."""
    a, b = cases["A"], cases["B"]
    assert not torch.equal(a["idx"], b["idx"]) and len(set(a["idx"].tolist()) & set(b["idx"].tolist())) < TC.N_RAYS // 4
    g = torch.Generator().manual_seed(0)
    assert torch.equal(a["idx"], torch.randperm(scene["ray_o"].shape[1], generator=g)[:TC.N_RAYS])
