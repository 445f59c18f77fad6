"""CPU: the tensor-core decoder keeps its wgmma chains pipelined on Hopper.

ptxas serialises every wgmma of a kernel (each one waits for the previous to finish) when it has to insert a warpgroup
arrive in a divergent path, and says so with the C7520 advisory.  The SASS then shows a WARPGROUP.DEPBAR after every HGMMA.
These tests compile the decoder for sm_90a and check both: no C7520, no register spills, and runs of back-to-back HGMMA
(one K-step of both N halves: 6 in the 3-pass mode, 2 in the 1-pass mode) with no DEPBAR between them."""
import os
import re
import shutil
import subprocess

import pytest

from neuralbody_b200 import _build

DECODER = "render_tc_list_kernel"


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    return exe


def _decoder_functions():
    txt = subprocess.run([_cuobjdump(), "-sass", _build.build()], capture_output=True, text=True, check=True).stdout
    out = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name, _, body = part.partition("\n")
        if DECODER in name:
            out[name.strip()] = body
    return out


def _longest_hgmma_run(body):
    best = cur = 0
    for line in body.splitlines():
        if re.search(r"\bHGMMA\.", line):
            cur += 1
            best = max(best, cur)
        elif "WARPGROUP.DEPBAR" in line or "WARPGROUP.ARRIVE" in line:
            cur = 0
    return best


def test_decoder_hgmma_issue_back_to_back():
    fns = _decoder_functions()
    assert len(fns) == 4, sorted(fns)            # <1 | 3 passes> x <fp32 | fp16 volume>
    for name, body in fns.items():
        need = 6 if "ILi3E" in name else 2
        assert _longest_hgmma_run(body) >= need, (name, _longest_hgmma_run(body))


def test_decoder_ptxas_no_serialisation_no_spills(tmp_path):
    src = os.path.join(_build.CSRC, "nb_render_tc_list.cu")
    cmd = [_build.find_nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "tcl.o"), src]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    assert "C7520" not in log, log
    # ptxas prints "Compiling entry function '<name>'", then its properties: stack frame, spill stores, registers
    entries = re.split(r"Compiling entry function '", log)[1:]
    dec = [e for e in entries if DECODER in e.split("'", 1)[0]]
    assert len(dec) == 4, log
    for e in dec:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m, e
        assert (int(m.group(1)), int(m.group(2))) == (0, 0), (e.split("'", 1)[0], m.group(0))
