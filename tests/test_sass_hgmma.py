"""CPU: the built library runs its tensor-core kernels on Hopper's warpgroup MMA (SASS of libneuralbody_b200.so, via
cuobjdump): the decoder and the training GEMM issue HGMMA for every K-step, so a refactor that silently drops them to a
generic path shows up without a GPU."""
import re
import shutil
import subprocess

import pytest

from neuralbody_b200 import _build


def _functions():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not shutil.os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    lib = _build.build()
    txt = subprocess.run([exe, "-sass", lib], capture_output=True, text=True, check=True).stdout
    assert "sm_90a" in txt
    out = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name, _, body = part.partition("\n")
        out[name.strip()] = body
    return out


def test_decoder_and_gemm_issue_hgmma():
    fns = _functions()
    dec = {n: b for n, b in fns.items() if "render_tc_list_kernel" in n}
    assert len(dec) == 4, sorted(dec)            # <1 | 3 passes> x <fp32 | fp16 volume>
    for name, body in dec.items():
        mma = len(re.findall(r"\bHGMMA\.64x128x16\.F32\b", body))
        l3 = len(re.findall(r"\bHGMMA\.64x64x16\.F32\b", body))
        # one push of a 256-wide layer = 2 K-steps x 2 N halves x (3 | 1) passes; layer 3 = 2 N halves per K-step
        assert mma >= (12 if "ILi3E" in name else 4), (name, mma)
        assert l3 >= 2, (name, l3)
        assert "UBLKCP" in body, name            # the weight stream arrives by bulk copy
    gemm = {n: b for n, b in fns.items() if "gemm_tf32x3_kernel" in n}
    assert len(gemm) == 4, sorted(gemm)
    for name, body in gemm.items():
        assert len(re.findall(r"\bHGMMA\.64x256x8\.F32\.TF32\b", body)) >= 3, name
