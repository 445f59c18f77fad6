"""The demo visualizers' frame and the rotate-SMPL drop-in without a GPU: the numpy restatement against the goldens and
(with the reference tree) the unmodified reference visualizers, the rotate drop-in's item against upstream's, the PNG
writer's ordering, error and exit semantics with fake events, nb_vis_frame's argument validation, and the drop-ins'
loading through the visualizer_module / visualizer_path factory."""
import ctypes as C
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from oracle import ref_harness
from oracle import vis_frames as O
from tools import demo_case as DC
from tools import vis_case as VC

needs_reference = pytest.mark.skipif(not ref_harness.reference_available(), reason="needs the reference tree")


@pytest.fixture(scope="module", autouse=True)
def _unload_reference():
    """The reference modules import the reference's `lib` package, which makes get_active_cfg() answer with the
    reference's cfg; take it out again after this module so later tests see this package's cfg."""
    before = set(sys.modules)
    yield
    for name in set(sys.modules) - before:
        if name == "lib" or name.startswith("lib.") or name in ("matplotlib", "matplotlib.pyplot", "termcolor", "PIL",
                                                                  "imageio", "plyfile", "trimesh"):
            del sys.modules[name]
    ref_harness._loaded = None


# ----------------------------------------------------------------------------- the restatement
def test_goldens_equal_the_restatement():
    g = VC.load_golden()
    assert set(g) == set(VC.CASES)
    for name, want in g.items():
        rgb, mask, (H, W, white) = VC.case(name)
        assert VC.checksum(rgb, mask) == bytes(want["sha256"]).decode(), name
        got = O.frame(rgb, mask, H, W, white)
        assert got.dtype == np.uint8 and got.shape == (H, W, 3) and np.array_equal(got, want["frame"]), name
    assert (g["empty"]["frame"] == 255).all()
    assert os.path.getsize(VC.GOLDEN) < 1 << 20


def test_the_cases_reach_what_they_are_for():
    rgb, mask, (H, W, _) = VC.case("border")
    m = mask.reshape(H, W)
    assert m[0].any() and m[:, 0].any() and m[:, -1].any()
    assert VC.case("empty")[0].shape == (0, 3)
    v = VC.case("saturate")[0]
    assert (v < 0).any() and (v > 1).any() and np.isnan(v).any() and (np.abs(v) * 255 > 2 ** 31).any()
    v = VC.case("ties")[0].astype(np.float64) * 255
    assert ((v % 1 == 0.5) & (v > 0) & (v < 255)).any() and (np.abs(v % 1 - 0.5) < 1e-4).sum() > 500


def test_restatement_raises_and_broadcasts_as_numpy():
    rgb, mask, (H, W, _) = VC.case("white")
    with pytest.raises(ValueError, match="cannot reshape"):
        O.frame(rgb, mask[:-1], H, W)
    with pytest.raises(ValueError, match="shape mismatch"):
        O.frame(rgb[:-1], mask, H, W)
    one = O.frame(rgb[:1], mask, H, W)          # a (1,3) value fills every set pixel, as numpy broadcasts it
    assert (one.reshape(-1, 3)[mask] == one.reshape(-1, 3)[mask][0]).all()


@needs_reference
@pytest.mark.parametrize("kind", ["demo", "perform"])
def test_restatement_writes_the_reference_visualizers_files(kind, tmp_path):
    cv2 = pytest.importorskip("cv2")
    cases = [VC.case(n) for n in ("white", "saturate", "ties", "empty")]
    rgb, mask = VC.random_view(70, 90, 3)
    cases.append((rgb, mask, (70, 90, 1)))
    for i, (rgb, mask, (H, W, white)) in enumerate(cases):
        want = VC.reference_png(kind, rgb, mask, H, W, white)
        p = str(tmp_path / ("%d.png" % i))
        assert cv2.imwrite(p, O.frame(rgb, mask, H, W, white))
        assert open(p, "rb").read() == want, i


@needs_reference
def test_reference_raises_where_the_restatement_does():
    rgb, mask, (H, W, white) = VC.case("white")
    for args in ((rgb[:-1], mask), (rgb, mask[:-1])):
        with pytest.raises(ValueError):
            VC.reference_png("demo", *args, H, W, white)
        with pytest.raises(ValueError):
            O.frame(*args, H, W, white)


# ----------------------------------------------------------------------------- the rotate-SMPL dataset
def test_rotate_golden_is_the_restatements_rays():
    """The golden's rays are image_rays of its camera and box (demo_case's restatement, pinned to upstream's own code), and
    its inputs are demo_case's synthetic tree."""
    g = VC.load_rotate_golden()
    for v, x in g["views"].items():
        got = DC.image_rays_numpy(x["RT"], x["K"], x["can_bounds"], g["H"], g["W"])
        for a, k in zip(got, ("ray_o", "ray_d", "near", "far", "mask_at_box")):
            assert np.array_equal(a, x[k]), (v, k)
        assert x["RT"].dtype == np.float64 and x["K"].dtype == np.float64 and x["can_bounds"].dtype == np.float32
        assert int(x["view_index"]) == v and int(x["frame_index"]) == 0
    boxes = [g["views"][v]["can_bounds"] for v in VC.ROTATE_VIEWS]
    assert not np.array_equal(boxes[0], boxes[1])          # the body turns with the view


def test_rotate_golden_inputs_are_rebuilt_without_the_reference(tmp_path):
    masks = DC.write_mv_root(str(tmp_path))
    assert DC.input_checksum(str(tmp_path), masks) == VC.load_rotate_golden()["input_sha256"]


@needs_reference
def test_rotate_drop_in_item_equals_upstreams(tmp_path):
    """The drop-in's item has every key of upstream's item but the rays, with upstream's values; its camera and box are
    what upstream hands image_rays; `meta` holds the same three."""
    from neuralbody_b200.lib.datasets.light_stage import rotate_smpl_dataset as drop
    views = (0, 5, 71, 143)
    pairs, _, ds, mod = VC.reference_rotate_items(views, str(tmp_path))
    cls = drop.make_dataset_class(mod.Dataset)
    mine = cls.__new__(cls)
    mine.__dict__.update(ds.__dict__)
    for v, (want, call) in zip(views, pairs):
        got = mine[v]
        rays = {"ray_o", "ray_d", "near", "far", "mask_at_box"}
        assert set(got) == (set(want) - rays) | {"cam_RT", "cam_K", "can_bounds", "meta"}
        for k in set(want) - rays:
            a, b = np.asarray(got[k]), np.asarray(want[k])
            assert a.dtype == b.dtype and np.array_equal(a, b), (v, k)
        for k, c in (("cam_RT", "RT"), ("cam_K", "K"), ("can_bounds", "bounds")):
            assert got[k].dtype == call[c].dtype and np.array_equal(got[k], call[c]), (v, k)
            assert got["meta"][k] is got[k]
    assert drop.Dataset is not None


# ----------------------------------------------------------------------------- the writer
class _FakeEvent:
    """Stands in for a torch.cuda.Event: synchronize() waits `delay` seconds and logs the call."""

    def __init__(self, log, name, delay=0.0):
        self.log, self.name, self.delay = log, name, delay

    def synchronize(self):
        time.sleep(self.delay)
        self.log.append(self.name)


def _visualizer(kind, monkeypatch, tmp_path, exp_name="exp"):
    import queue
    from neuralbody_b200.lib.config import cfg, get_active_cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    monkeypatch.chdir(tmp_path)
    monkeypatch.setitem(get_active_cfg(), "exp_name", exp_name)
    path = cfg.visualizer_path.replace("if_nerf_demo", "if_nerf_" + kind)
    vis = load_source(cfg.visualizer_module.replace("if_nerf_demo", "if_nerf_" + kind), path).Visualizer()
    vis._free = queue.Queue()
    return vis


def _slot(frame, fi, vi, n, status=0, count=None):
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.visualizers.frame_writer import Slot
    H, W = frame.shape[:2]
    s = Slot(H, W, pin=False)
    r = capi.nb_vis_frame_result(status, n if count is None else count)
    s.out.numpy()[:C.sizeof(r)] = np.frombuffer(bytes(r), np.uint8)
    s.out.numpy()[256:] = frame.reshape(-1)
    s.idx.numpy()[:] = (fi, vi)
    s.n = n
    return s


def test_writer_order_errors_and_flush(monkeypatch, tmp_path):
    cv2 = pytest.importorskip("cv2")
    vis = _visualizer("demo", monkeypatch, tmp_path)
    log = []
    rng = np.random.RandomState(0)
    frames = [rng.randint(0, 256, (12, 10, 3)).astype(np.uint8) for _ in range(6)]
    slots = []
    for i, f in enumerate(frames):
        s = _slot(f, 2, i, 5)
        s.event = _FakeEvent(log, i, 0.05 if i == 0 else 0.0)
        slots.append(s)
        vis._enqueue(s, "exp")
    vis.flush()
    assert log == list(range(6))               # one thread, in order, each after its event
    for i, f in enumerate(frames):
        p = tmp_path / "data" / "render" / "exp" / "frame_0002" / ("%04d.png" % i)
        assert np.array_equal(cv2.imread(str(p), cv2.IMREAD_UNCHANGED), f)
    assert vis._free.qsize() == 6              # every slot is free again
    # a count mismatch is raised by the next flush(); the views queued after it are not written
    bad = _slot(frames[0], 3, 0, 5, status=1, count=7)
    bad.event = _FakeEvent(log, "bad")
    after = _slot(frames[1], 3, 1, 5)
    after.event = _FakeEvent(log, "after")
    vis._enqueue(bad, "exp")
    vis._enqueue(after, "exp")
    with pytest.raises(ValueError, match=r"shape mismatch: value array of shape \(5,3\).*\(7,3\)"):
        vis.flush()
    assert not (tmp_path / "data" / "render" / "exp" / "frame_0003").exists() and "after" not in log
    assert vis._free.qsize() == 8
    vis.flush()                                # the error was raised once
    # ... and by the next visualize(), before it reads anything
    vis._enqueue(_slot(frames[0], 4, 0, 5, status=1, count=4), "exp")
    vis._writer._q.join()
    with pytest.raises(ValueError, match="shape mismatch"):
        vis.visualize({}, {})


def test_perform_paths(monkeypatch, tmp_path):
    pytest.importorskip("cv2")
    vis = _visualizer("perform", monkeypatch, tmp_path, "pexp")
    vis._enqueue(_slot(np.zeros((4, 6, 3), np.uint8), 12, 3, 1), "pexp")
    vis.flush()
    assert (tmp_path / "data" / "perform" / "pexp" / "0" / "frame0012_view0003.png").is_file()
    from neuralbody_b200.lib.visualizers import if_nerf_demo
    for kind, v in (("perform", vis), ("demo", if_nerf_demo.Visualizer())):
        assert v.frame_path("e", 12, 3) == VC.reference_path(kind, "e", 12, 3)


def test_writer_raises_when_imwrite_fails(monkeypatch):
    """Upstream ignores a False from cv2.imwrite; the writer raises IOError."""
    import types
    from neuralbody_b200.png_writer import PngWriter
    monkeypatch.setitem(sys.modules, "cv2", types.SimpleNamespace(imwrite=lambda p, img: False))
    done = threading.Event()
    w = PngWriter()
    w.submit(("nowhere.png", np.zeros((2, 2, 3), np.uint8)), done=done.set)
    with pytest.raises(IOError, match="nowhere.png"):
        w.join()
    assert done.is_set()


def test_queued_views_reach_the_disk_at_exit(tmp_path):
    """A process that queues views and exits without flush(): the atexit handler writes them all."""
    pytest.importorskip("cv2")
    from conftest import ROOT
    script = """
import sys, queue, time
sys.path.insert(0, %r)
import numpy as np
sys.path.insert(0, %r)
from test_vis_frames_cpu import _slot, _FakeEvent
from neuralbody_b200.lib.config import cfg
from neuralbody_b200.lib.visualizers import if_nerf_demo
cfg.exp_name = "atexit"
vis = if_nerf_demo.Visualizer()
vis._free = queue.Queue()
log = []
for i in range(5):
    s = _slot(np.full((8, 8, 3), i, np.uint8), 1, i, 3)
    s.event = _FakeEvent(log, i, 0.3)
    vis._enqueue(s, "atexit")
print("queued", len(log))
""" % (ROOT, os.path.join(ROOT, "tests"))
    res = subprocess.run([sys.executable, "-c", script], cwd=str(tmp_path), capture_output=True, text=True, timeout=120)
    assert res.returncode == 0, res.stderr
    assert "queued 0" in res.stdout                   # nothing was written when the script's last line ran
    d = tmp_path / "data" / "render" / "atexit" / "frame_0001"
    assert sorted(os.listdir(d)) == ["%04d.png" % i for i in range(5)]


# ----------------------------------------------------------------------------- the C ABI and the factory
def test_c_abi_validates_its_arguments(built_lib):
    """Every check fails before anything is enqueued (the pointers below are not device memory)."""
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_vis_frame_workspace_bytes(0, 512) == 0
    assert lib.nb_vis_frame_workspace_bytes(512, -1) == 0
    assert lib.nb_vis_frame_workspace_bytes(65536, 65536) == 0
    ws = lib.nb_vis_frame_workspace_bytes(16, 16) or 1 << 20    # the CUB size query needs a device

    def args(**kw):
        a = capi.nb_vis_frame_args()
        a.n, a.H, a.W = 10, 16, 16
        a.rgb_map = a.mask_at_box = a.workspace = a.result = a.frame = 256
        a.workspace_bytes = ws
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for kw, what in (({"mask_at_box": None}, b"null"), ({"rgb_map": None}, b"null"), ({"result": None}, b"null"),
                     ({"frame": None}, b"null"), ({"workspace": None}, b"null"), ({"H": 0}, b"H, W"),
                     ({"W": 70000, "H": 70000}, b"H, W"), ({"n": -1}, b"H, W"), ({"n": 1 << 30}, b"H, W"),
                     ({"white_bkgd": 2}, b"white_bkgd"), ({"frame": 258}, b"aligned"),
                     ({"workspace_bytes": ws - 1}, b"workspace")):
        assert lib.nb_vis_frame(C.byref(args(**kw)), None) == -1, kw   # NB_ERR_BAD_ARG
        err = lib.nb_last_error()
        assert b"nb_vis_frame" in err and what in err, (kw, err)
    assert lib.nb_vis_frame(None, None) == -1


def test_result_layout_matches_the_header(built_lib):
    from conftest import ROOT
    from neuralbody_b200 import capi
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "neuralbody_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
           'sizeof(nb_vis_frame_result), sizeof(nb_vis_frame_args), offsetof(nb_vis_frame_args, rgb_map), '
           'offsetof(nb_vis_frame_args, frame));return 0;}\n')
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "p")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(capi.nb_vis_frame_result), C.sizeof(capi.nb_vis_frame_args),
                     capi.nb_vis_frame_args.rgb_map.offset, capi.nb_vis_frame_args.frame.offset]


def test_drop_ins_load_through_the_factory_with_upstreams_keys(capsys):
    """make_visualizer.py:5-9: imp.load_source(cfg.visualizer_module, cfg.visualizer_path).Visualizer() prints upstream's
    line; a batch without view_index is upstream's KeyError, raised before anything runs on the device."""
    import torch
    from neuralbody_b200.lib.config import cfg, get_active_cfg
    from neuralbody_b200.lib.config.config import _defaults
    from neuralbody_b200.lib.networks.make_network import load_source
    d = _defaults()
    assert d.visualizer_module == cfg.visualizer_module == "neuralbody_b200.lib.visualizers.if_nerf_demo"
    assert os.path.isfile(d.visualizer_path)
    vis = load_source(cfg.visualizer_module, cfg.visualizer_path).Visualizer()
    active = get_active_cfg()         # the reference's, while the tests above have its `lib` loaded
    assert "the results are saved at data/render/%s" % active.exp_name in capsys.readouterr().out
    H, W = int(active.H * active.ratio), int(active.W * active.ratio)
    with pytest.raises(KeyError):
        vis.visualize({"rgb_map": torch.zeros((1, 0, 3))}, {"mask_at_box": torch.zeros((1, H * W), dtype=torch.bool),
                                                             "frame_index": torch.tensor([0])})
    with pytest.raises(ValueError, match="cannot reshape array of size 5"):
        vis.visualize({"rgb_map": torch.zeros((1, 0, 3))}, {"mask_at_box": torch.zeros((1, 5), dtype=torch.bool)})
    from neuralbody_b200.lib.visualizers import if_nerf_perform
    if_nerf_perform.Visualizer()
    assert "the results are saved at data/perform/%s" % active.exp_name in capsys.readouterr().out
