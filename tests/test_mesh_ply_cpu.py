"""The mesh mode's PLY path without a GPU: ply_header plus a numpy restatement of nb_mesh_ply's body against Mesh.export's
bytes, nb_mesh_ply's host-side rejections and struct layout, the mesh visualizer drop-in's naming, order, errors, flush(),
exit drain and back-pressure with host meshes and fake events, its loading through the visualizer_module /
visualizer_path factory, and the renderer's mesh_output validation."""
import ctypes as C
import io
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

from conftest import ROOT

MESH_VISUALIZER = os.path.join(ROOT, "neuralbody_b200", "lib", "visualizers", "if_nerf_mesh.py")
MESH_RENDERER = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")


def ply_body(vertices, faces):
    """nb_mesh_ply's body, restated: the vertices' float64 bytes, then per face uchar 3 and three little-endian int32."""
    v = np.ascontiguousarray(vertices, dtype="<f8").reshape(-1, 3)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    rec = np.empty((len(f), 13), np.uint8)
    rec[:, 0] = 3
    rec[:, 1:] = f.astype("<i4").view(np.uint8).reshape(-1, 12)
    return v.tobytes() + rec.tobytes()


def random_mesh(nv, nf, seed):
    rng = np.random.RandomState(seed)
    return rng.randn(nv, 3) * 50, rng.randint(0, max(nv, 1), (nf, 3)).astype(np.int64)


# ----------------------------------------------------------------------------- the bytes
@pytest.mark.parametrize("nv,nf", [(0, 0), (1, 0), (1, 1), (3, 1), (31, 33), (32, 31), (33, 32), (1001, 1999)])
def test_header_and_restated_body_equal_mesh_export(nv, nf):
    from neuralbody_b200 import mcubes
    v, f = random_mesh(nv, nf, nv * 7 + nf)
    buf = io.BytesIO()
    data = mcubes.Mesh(v, f).export(buf)
    assert buf.getvalue() == data == mcubes.ply_header(nv, nf) + ply_body(v, f)
    assert len(ply_body(v, f)) == 24 * nv + 13 * nf


def test_header_text():
    from neuralbody_b200 import mcubes
    assert mcubes.ply_header(7, 5) == (b"ply\nformat binary_little_endian 1.0\nelement vertex 7\nproperty double x\n"
                                       b"property double y\nproperty double z\nelement face 5\n"
                                       b"property list uchar int vertex_indices\nend_header\n")


def test_restatement_keeps_special_vertex_bits_and_extreme_indices(tmp_path):
    from neuralbody_b200 import mcubes
    v = np.array([[-0.0, np.nan, np.inf], [-np.inf, 5e-324, -2.2250738585072014e-308], [1.0, -1.0, 0.0]])
    f = np.array([[0, 2, 1], [2, 2, 0]], np.int64)
    p = str(tmp_path / "m.ply")
    mcubes.Mesh(v, f).export(p)
    assert open(p, "rb").read() == mcubes.ply_header(3, 2) + ply_body(v, f)
    rv, rf = mcubes.read_ply(p)
    assert np.array_equal(rv.view(np.int64), v.view(np.int64)) and np.array_equal(rf, f)


# ----------------------------------------------------------------------------- the C ABI
def test_c_abi_validates_its_arguments(built_lib):
    """Every check fails before anything is enqueued (the pointers below are not device memory)."""
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_mesh_ply_bytes(0, 0) == 0
    assert lib.nb_mesh_ply_bytes(5, 7) == 24 * 5 + 13 * 7
    assert lib.nb_mesh_ply_bytes((1 << 31) - 1, 3) == 24 * ((1 << 31) - 1) + 39
    for nv, nf in ((-1, 0), (0, -1), (1 << 31, 0), (0, (1 << 40) + 1)):
        assert lib.nb_mesh_ply_bytes(nv, nf) == 0, (nv, nf)

    def args(**kw):
        a = capi.nb_mesh_ply_args()
        a.nv, a.nf = 10, 12
        a.vertices = a.faces = a.out = 256
        a.out_bytes = 16 + 24 * 10 + 13 * 12
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for kw, what in (({"out": None}, b"null"), ({"vertices": None}, b"null"), ({"faces": None}, b"null"),
                     ({"nv": -1}, b"counts"), ({"nf": -3}, b"counts"), ({"nf": (1 << 40) + 1}, b"counts"),
                     ({"nv": 1 << 31, "nf": 0}, b"2^31"), ({"nv": 1 << 33}, b"2^31"),
                     ({"out": 264}, b"aligned"), ({"vertices": 260}, b"aligned"), ({"faces": 252}, b"aligned"),
                     ({"out_bytes": 16 + 24 * 10 + 13 * 12 - 1}, b"out_bytes"), ({"out_bytes": 24 * 10 + 13 * 12}, b"out_bytes")):
        assert lib.nb_mesh_ply(C.byref(args(**kw)), None) == -1, kw   # NB_ERR_BAD_ARG
        err = lib.nb_last_error()
        assert b"nb_mesh_ply" in err and what in err, (kw, err)
    assert lib.nb_mesh_ply(None, None) == -1


def test_struct_layout_matches_the_header(built_lib):
    from neuralbody_b200 import capi
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "neuralbody_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu '
           '%d %d %d\\n", sizeof(nb_mesh_ply_result), sizeof(nb_mesh_ply_args), offsetof(nb_mesh_ply_args, vertices), '
           'offsetof(nb_mesh_ply_args, out), offsetof(nb_mesh_ply_args, out_bytes), NB_MESH_PLY_BODY_OFFSET, '
           'NB_MESH_PLY_OK, NB_MESH_PLY_FACE);return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "p")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(capi.nb_mesh_ply_result), C.sizeof(capi.nb_mesh_ply_args), capi.nb_mesh_ply_args.vertices.offset,
                   capi.nb_mesh_ply_args.out.offset, capi.nb_mesh_ply_args.out_bytes.offset, capi.NB_MESH_PLY_BODY_OFFSET,
                   capi.NB_MESH_PLY_OK, capi.NB_MESH_PLY_FACE]
    assert C.sizeof(capi.nb_mesh_ply_result) <= capi.NB_MESH_PLY_BODY_OFFSET


# ----------------------------------------------------------------------------- the visualizer
class _FakeEvent:
    """Stands in for a torch.cuda.Event: synchronize() waits `delay` seconds and logs the call."""

    def __init__(self, log, name, delay=0.0):
        self.log, self.name, self.delay = log, name, delay

    def synchronize(self):
        time.sleep(self.delay)
        self.log.append(self.name)


class _GatedMesh:
    """A host mesh whose export logs its path and waits for `gate` before writing a Mesh's file."""

    def __init__(self, mesh, log, gate=None):
        self.mesh, self.log, self.gate = mesh, log, gate

    def export(self, path):
        if self.gate is not None:
            self.gate.wait(30)
        self.log.append(os.path.basename(path))
        return self.mesh.export(path)


def _visualizer(monkeypatch, tmp_path, result_dir="res"):
    from neuralbody_b200.lib.config import get_active_cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    cfg = get_active_cfg()
    monkeypatch.chdir(tmp_path)
    monkeypatch.setitem(cfg, "result_dir", result_dir)
    monkeypatch.setitem(cfg, "visualizer_module", "neuralbody_b200.lib.visualizers.if_nerf_mesh")
    monkeypatch.setitem(cfg, "visualizer_path", MESH_VISUALIZER)
    return load_source(cfg.visualizer_module, cfg.visualizer_path).Visualizer()


def _device_slot(v, f, fi, status=0):
    """A filled slot as a DeviceMesh frame leaves it: the status record and the restated body, frame_index."""
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.visualizers.if_nerf_mesh import MeshSlot
    s = MeshSlot(pin=False)
    body = ply_body(v, f)
    out = s.reserve(capi.NB_MESH_PLY_BODY_OFFSET + len(body)).numpy()
    out[:] = 0
    out[:C.sizeof(capi.nb_mesh_ply_result)] = np.frombuffer(bytes(capi.nb_mesh_ply_result(status)), np.uint8)
    out[capi.NB_MESH_PLY_BODY_OFFSET:] = np.frombuffer(body, np.uint8)
    s.nv, s.nf = len(v), len(f)
    s.idx.numpy()[0] = fi
    return s


def test_paths_directory_and_host_meshes(monkeypatch, tmp_path, capsys):
    import torch
    from neuralbody_b200 import mcubes
    vis = _visualizer(monkeypatch, tmp_path, "out/r")
    assert "the results are saved at out/r/mesh" in capsys.readouterr().out
    meshes = [mcubes.Mesh(*random_mesh(20 + i, 30 + i, i)) for i in range(3)]
    for fi, m in zip((7, 12345, 0), meshes):
        vis.visualize({"mesh": m, "cube": None}, {"frame_index": torch.tensor([fi])})
    vis.flush()
    d = tmp_path / "out" / "r" / "mesh"
    assert sorted(os.listdir(d)) == ["0000.ply", "0007.ply", "12345.ply"]
    for fi, m in zip((7, 12345, 0), meshes):
        assert (d / ("%04d.ply" % fi)).read_bytes() == m.export(io.BytesIO())
    assert vis._free.qsize() == 4 and all(s.mesh is None for s in list(vis._free.queue))


def test_device_slots_order_errors_and_flush(monkeypatch, tmp_path):
    from neuralbody_b200 import mcubes
    vis = _visualizer(monkeypatch, tmp_path)
    d = os.path.join("res", "mesh")
    log = []
    meshes = [random_mesh(n, n + 3, n) for n in (0, 1, 33, 64)]
    for i, (v, f) in enumerate(meshes):
        vis._free.get()
        vis._enqueue(_device_slot(v, f, i), d, _FakeEvent(log, i, 0.05 if i == 0 else 0.0))
    vis.flush()
    assert log == [0, 1, 2, 3]                 # one thread, in order, each after its event
    for i, (v, f) in enumerate(meshes):
        assert (tmp_path / d / ("%04d.ply" % i)).read_bytes() == mcubes.Mesh(v, f).export(io.BytesIO())
    # a face-range status is raised by the next flush(); that frame and the ones queued after it are not written
    v, f = random_mesh(5, 4, 1)
    vis._enqueue(_device_slot(v, f, 10, status=1), d, _FakeEvent(log, "bad"))
    vis._enqueue(_device_slot(v, f, 11), d, _FakeEvent(log, "after"))
    with pytest.raises(ValueError, match="face indices out of range"):
        vis.flush()
    assert not (tmp_path / d / "0010.ply").exists() and not (tmp_path / d / "0011.ply").exists()
    assert "after" not in log
    vis.flush()                                # the error was raised once
    # ... and by the next visualize(), before it reads anything
    vis._enqueue(_device_slot(v, f, 12, status=1), d, None)
    vis._writer._q.join()
    with pytest.raises(ValueError, match="face indices out of range"):
        vis.visualize({}, {})


def test_host_mesh_error_and_writer_order(monkeypatch, tmp_path):
    import torch
    from neuralbody_b200 import mcubes
    vis = _visualizer(monkeypatch, tmp_path)
    log = []
    good = mcubes.Mesh(*random_mesh(6, 5, 3))
    bad = mcubes.Mesh(np.zeros((2, 3)), np.array([[0, 1, 2]]))
    for fi, m in ((1, good), (2, bad), (3, good)):
        vis.visualize({"mesh": _GatedMesh(m, log)}, {"frame_index": torch.tensor([fi])})
    with pytest.raises(ValueError, match="face indices out of range"):
        vis.flush()
    assert log == ["0001.ply", "0002.ply"]
    assert sorted(os.listdir(tmp_path / "res" / "mesh")) == ["0001.ply"]
    assert vis._free.qsize() == 4


def test_back_pressure_at_four_slots(monkeypatch, tmp_path):
    import torch
    from neuralbody_b200 import mcubes
    from neuralbody_b200.lib.visualizers import if_nerf_mesh
    assert if_nerf_mesh.SLOTS == 4
    vis = _visualizer(monkeypatch, tmp_path)
    log, gate = [], threading.Event()
    m = mcubes.Mesh(*random_mesh(4, 2, 0))
    returned = []

    def loop():
        for fi in range(6):
            vis.visualize({"mesh": _GatedMesh(m, log, gate)}, {"frame_index": fi})
            returned.append(fi)

    th = threading.Thread(target=loop, daemon=True)
    th.start()
    time.sleep(0.5)
    assert returned == [0, 1, 2, 3] and log == []      # four frames hold the four slots; the fifth waits for one
    gate.set()
    th.join(30)
    assert returned == list(range(6))
    vis.flush()
    assert log == ["%04d.ply" % i for i in range(6)]


def test_queued_frames_reach_the_disk_at_exit(tmp_path):
    """A process that queues frames and exits without flush(): the atexit handler writes them all."""
    script = """
import sys, time
sys.path.insert(0, %r)
sys.path.insert(0, %r)
from test_mesh_ply_cpu import _device_slot, _FakeEvent, random_mesh
from neuralbody_b200.lib.config import cfg
from neuralbody_b200.lib.visualizers import if_nerf_mesh
cfg.result_dir = "atexit"
vis = if_nerf_mesh.Visualizer()
log = []
for i in range(4):
    vis._free.get()
    vis._enqueue(_device_slot(*random_mesh(9, 8, i), i), "atexit/mesh", _FakeEvent(log, i, 0.3))
print("queued", len(log))
""" % (ROOT, os.path.join(ROOT, "tests"))
    res = subprocess.run([sys.executable, "-c", script], cwd=str(tmp_path), capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    assert "queued 0" in res.stdout                   # nothing was written when the script's last line ran
    d = tmp_path / "atexit" / "mesh"
    assert sorted(os.listdir(d)) == ["%04d.ply" % i for i in range(4)]
    from neuralbody_b200 import mcubes
    assert (d / "0002.ply").read_bytes() == mcubes.Mesh(*random_mesh(9, 8, 2)).export(io.BytesIO())


def test_slot_buffer_is_replaced_only_when_too_small():
    from neuralbody_b200.lib.visualizers.if_nerf_mesh import MeshSlot
    s = MeshSlot(pin=False)
    a = s.reserve(1000)
    first = s.out
    assert a.numel() == 1000 and first.numel() >= 1000
    assert s.reserve(900).numel() == 900 and s.out is first
    assert s.reserve(first.numel()).numel() == first.numel() and s.out is first
    s.reserve(first.numel() + 1)
    assert s.out is not first and s.out.numel() > first.numel()


# ----------------------------------------------------------------------------- the factory and the renderer's key
def test_drop_in_loads_through_the_factory(monkeypatch, tmp_path, capsys):
    from neuralbody_b200.lib.config import get_active_cfg
    vis = _visualizer(monkeypatch, tmp_path, "data/result/if_nerf/x")
    assert "the results are saved at data/result/if_nerf/x/mesh" in capsys.readouterr().out
    assert hasattr(vis, "visualize") and hasattr(vis, "flush")
    with pytest.raises(KeyError):
        vis.visualize({}, {"frame_index": 0})
    assert vis._free.qsize() == 4
    assert get_active_cfg().result_dir == "data/result/if_nerf/x"


def test_mesh_output_validation(built_lib, monkeypatch):
    from neuralbody_b200.lib.config import get_active_cfg
    from neuralbody_b200.lib.config.config import _defaults
    from neuralbody_b200.lib.networks.make_network import load_source
    mod = load_source("neuralbody_b200.lib.networks.renderer.if_mesh_renderer", MESH_RENDERER)
    assert _defaults().mesh_output == "host" and mod.MESH_OUTPUTS == ("host", "device")
    cfg = get_active_cfg()
    assert mod.mesh_output({}) == "host"                 # upstream's cfg has no such key
    for m in mod.MESH_OUTPUTS:
        assert mod.mesh_output({"mesh_output": m}) == m
    r = mod.Renderer.__new__(mod.Renderer)
    for bad in ("cpu", "Device", None, 1):
        monkeypatch.setitem(cfg, "mesh_output", bad)
        with pytest.raises(ValueError, match="'host', 'device'"):
            r.render({})                                  # raised before anything else runs
