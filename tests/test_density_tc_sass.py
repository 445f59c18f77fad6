"""CPU: the density-only tensor-core decoder (density_tc_list_kernel, nb_decode_density_list) is built like the render
decoder: four <passes, volume dtype> instantiations, no C7520 serialisation advisory, no register spills, and runs of
back-to-back HGMMA (6 per K-step in the 3-pass mode, 2 in the 1-pass mode) with no warpgroup wait between them."""
import os
import re
import subprocess

from neuralbody_b200 import _build
from test_decoder_wgmma_pipeline import _cuobjdump, _longest_hgmma_run

DENSITY = "density_tc_list_kernel"


def test_density_decoder_hgmma_issue_back_to_back():
    txt = subprocess.run([_cuobjdump(), "-sass", _build.build()], capture_output=True, text=True, check=True).stdout
    fns = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name, _, body = part.partition("\n")
        if DENSITY in name:
            fns[name.strip()] = body
    assert len(fns) == 4, sorted(fns)            # <1 | 3 passes> x <fp32 | fp16 volume>
    for name, body in fns.items():
        need = 6 if "ILi3E" in name else 2
        assert _longest_hgmma_run(body) >= need, (name, _longest_hgmma_run(body))
        assert not re.search(r"\bHGMMA\.64x64x16", body), name          # no layer 3 (the colour layer)


def test_density_decoder_ptxas_no_serialisation_no_spills(tmp_path):
    src = os.path.join(_build.CSRC, "nb_render_tc_list.cu")
    cmd = [_build.find_nvcc()] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", "-o", str(tmp_path / "tcl.o"), src]
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    assert "C7520" not in log, log
    entries = re.split(r"Compiling entry function '", log)[1:]
    dec = [e for e in entries if DENSITY in e.split("'", 1)[0]]
    assert len(dec) == 4, log
    for e in dec:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", e)
        assert m, e
        assert (int(m.group(1)), int(m.group(2))) == (0, 0), (e.split("'", 1)[0], m.group(0))
