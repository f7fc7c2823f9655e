"""CPU-side checks of the CUDA-graph path: rgs_forward_preset's host rejections (before any CUDA call), the capacity rule of
rade_gs_b200.graphs.BinningReserve, and StepGraph's keys, LRU bound and overflow fallback with the step and the graph stubbed."""
import ctypes
import os

import pytest
import torch

from conftest import ROOT

LIB = os.path.join(ROOT, "rade-gs_b200", "rade_gs_b200", "librgs_b200.so")


class Cam(ctypes.Structure):
    _fields_ = [("width", ctypes.c_int32), ("height", ctypes.c_int32), ("tan_fovx", ctypes.c_float), ("tan_fovy", ctypes.c_float),
                ("kernel_size", ctypes.c_float), ("scale_modifier", ctypes.c_float), ("viewmatrix", ctypes.c_void_p), ("projmatrix", ctypes.c_void_p),
                ("cam_pos", ctypes.c_void_p), ("background", ctypes.c_void_p), ("sh_degree", ctypes.c_int32), ("sh_coeffs", ctypes.c_int32),
                ("require_coord", ctypes.c_int32), ("require_depth", ctypes.c_int32), ("prefiltered", ctypes.c_int32), ("debug", ctypes.c_int32),
                ("tile_row_begin", ctypes.c_int32), ("tile_row_end", ctypes.c_int32), ("compact_slab", ctypes.c_int32)]


class Gs(ctypes.Structure):
    _fields_ = [("P", ctypes.c_int32)] + [(n, ctypes.c_void_p) for n in ("means3D", "opacities", "shs", "colors_precomp", "scales", "rotations",
                                                                         "cov3D_precomp", "shs_rest")]


class Preset(ctypes.Structure):
    _fields_ = [("instances", ctypes.c_int64), ("longest_list", ctypes.c_int32), ("status", ctypes.c_void_p)]


FAKE = ctypes.c_void_p(0x1000)   # never dereferenced: every case below is rejected before the first CUDA call


def _lib():
    lib = ctypes.CDLL(LIB)
    lib.rgs_last_error.restype = ctypes.c_char_p
    lib.rgs_forward_preset.restype = ctypes.c_int64
    return lib


def _call(lib, preset="default", **cam_fields):
    cam = Cam(width=64, height=64, tan_fovx=0.5, tan_fovy=0.5, scale_modifier=1.0, sh_degree=3, sh_coeffs=16, tile_row_begin=0, tile_row_end=-1)
    for k, v in cam_fields.items():
        setattr(cam, k, v)
    gs = Gs(P=4, means3D=FAKE, opacities=FAKE, shs=FAKE, scales=FAKE, rotations=FAKE)
    out = (ctypes.c_void_p * 8)(*[FAKE] * 8)
    bufs = (ctypes.c_void_p * 6)(*[FAKE] * 6)
    if preset == "default":
        preset = Preset(instances=1 << 16, longest_list=256, status=FAKE)
    p = ctypes.byref(preset) if preset is not None else None
    return lib.rgs_forward_preset(ctypes.byref(cam), ctypes.byref(gs), out, bufs, p, None), lib.rgs_last_error()


@pytest.mark.parametrize("case, code, words", [
    ("null preset", -1, b"null preset"),
    ("null status", -1, b"null preset / status"),
    ("negative instances", -1, b"negative capacity"),
    ("negative list", -1, b"negative capacity"),
    ("debug", -3, b"debug"),
    ("slab", -3, b"whole image"),
    ("slab end", -3, b"whole image"),
    ("compact", -3, b"whole image"),
    ("prefiltered", -3, b"prefiltered"),
])
def test_forward_preset_host_rejections(case, code, words):
    lib = _lib()
    preset, cam = "default", {}
    if case == "null preset":
        preset = None
    elif case == "null status":
        preset = Preset(instances=1 << 16, longest_list=256, status=None)
    elif case == "negative instances":
        preset = Preset(instances=-1, longest_list=256, status=FAKE)
    elif case == "negative list":
        preset = Preset(instances=1 << 16, longest_list=-1, status=FAKE)
    elif case == "debug":
        cam = {"debug": 1}
    elif case == "slab":
        cam = {"tile_row_begin": 1, "tile_row_end": 3}
    elif case == "slab end":
        cam = {"tile_row_end": 4}
    elif case == "compact":
        cam = {"compact_slab": 1}
    elif case == "prefiltered":
        cam = {"prefiltered": 1}
    rc, msg = _call(lib, preset, **cam)
    assert rc == code and words in msg, (rc, msg)


def test_forward_preset_checks_the_frame_like_rgs_forward():
    rc, msg = _call(_lib(), sh_coeffs=20)
    assert rc == -1 and b"at most 16 SH coefficients" in msg
    lib = _lib()
    assert lib.rgs_forward_preset(None, None, None, None, None, None) == -1


# ---- BinningReserve ---------------------------------------------------------------------------------------------------

def test_reserve_fitting_rule():
    from rade_gs_b200.graphs import BinningReserve
    r = BinningReserve("cpu")
    assert (r.instances, r.longest_list) == (0, 0)
    assert r.status.dtype == torch.int32 and r.status.shape == (4,)
    assert not r.fit(0, 0)
    assert r.fit(1, 1) and (r.instances, r.longest_list) == (65536, 256)
    assert not r.fit(52428, 204), "52428 * 5/4 = 65535 and 204 * 5/4 = 255 fit the capacities"


def test_reserve_fitting_rule_exact_values():
    from rade_gs_b200.graphs import BinningReserve
    cases = [((52428, 204), (65536, 256)),        # 65535 and 255 fit the first granule
             ((52429, 205), (131072, 512)),       # 65537 (rounded up from 65536.25) and 257 (256.25) need the next
             ((800_000, 3000), (1_048_576, 3840)),
             ((1, 8193), (65536, 10496))]
    for (inst, lst), want in cases:
        r = BinningReserve("cpu")
        r.fit(inst, lst)
        assert (r.instances, r.longest_list) == want, (inst, lst)
    r = BinningReserve("cpu", 1 << 20, 4096)
    assert (r.instances, r.longest_list) == (1_310_720, 5120)
    assert not r.fit(10, 10), "never shrinks"
    assert (r.instances, r.longest_list) == (1_310_720, 5120)
    with pytest.raises(ValueError):
        r.fit(-1, 0)


def test_reserve_status_read_and_growth():
    from rade_gs_b200.graphs import BinningReserve
    r = BinningReserve("cpu", 65536, 256)
    assert not r.overflowed()
    r.status.copy_(torch.tensor([2, 70000, 300, 0], dtype=torch.int32))
    assert r.read() == (2, 70000, 300)
    assert r.overflowed()
    assert (r.instances, r.longest_list) == (131072, 512)
    r.status.copy_(torch.tensor([0, 100, 10, 0], dtype=torch.int32))
    assert not r.overflowed() and (r.instances, r.longest_list) == (131072, 512), "no growth without an overflow bit"
    r.status.copy_(torch.tensor([1, -1, 5, 0], dtype=torch.int32))   # the device words are unsigned
    assert r.read() == (1, 0xFFFFFFFF, 5)
    r.clear()
    assert r.status.tolist() == [0, 0, 0, 0]


# ---- StepGraph with the step and the graph stubbed ----------------------------------------------------------------------

class _StubReserve:
    def __init__(self):
        self.script = []
        self.reads = 0

    def overflowed(self):
        self.reads += 1
        return self.script.pop(0) if self.script else False


class _StubGraph:
    def __init__(self, key, log):
        self.key, self.log = key, log

    def replay(self):
        self.log.append(("replay", self.key))
        return ("graph", self.key)


@pytest.fixture
def stepgraph(monkeypatch):
    from rade_gs_b200 import graphs
    log = []
    current = {}

    def capture(self, fn, params):
        log.append(("capture", current["key"]))
        return _StubGraph(current["key"], log)

    monkeypatch.setattr(graphs.StepGraph, "_capture", capture)

    def make(max_graphs=4):
        sg = graphs.StepGraph(_StubReserve(), max_graphs=max_graphs)

        def run(key, params=()):
            current["key"] = key

            def fn():
                log.append(("eager", key))
                return ("eager", key)
            return sg.run(key, fn, params)
        return sg, run, log
    return make


def test_stepgraph_captures_once_per_key_and_replays(stepgraph):
    sg, run, log = stepgraph()
    assert run("a") == ("graph", "a")
    assert run("a") == ("graph", "a")
    assert run("b") == ("graph", "b")
    assert log == [("capture", "a"), ("replay", "a"), ("replay", "a"), ("capture", "b"), ("replay", "b")]
    assert sg.captures == 2 and len(sg) == 2 and "a" in sg
    assert sg.reserve.reads == 3, "one status read per step"


def test_stepgraph_lru_bound(stepgraph):
    sg, run, log = stepgraph(max_graphs=2)
    run("a")
    run("b")
    run("a")          # a is now the most recent
    run("c")          # evicts b
    assert "a" in sg and "c" in sg and "b" not in sg and len(sg) == 2
    log.clear()
    run("b")          # recaptured, evicts a
    assert log[0] == ("capture", "b") and "a" not in sg and len(sg) == 2
    with pytest.raises(ValueError):
        from rade_gs_b200.graphs import StepGraph
        StepGraph(_StubReserve(), max_graphs=0)


def test_stepgraph_overflow_runs_the_step_eagerly_and_recaptures(stepgraph):
    sg, run, log = stepgraph()
    p = torch.ones(3, requires_grad=True)
    p.grad = torch.full((3,), 7.0)
    grad = p.grad
    run("a", [p])
    run("b", [p])
    sg.reserve.script = [True]
    log.clear()
    assert run("a", [p]) == ("eager", "a")
    assert log == [("replay", "a"), ("eager", "a")]
    assert p.grad is grad and bool((p.grad == 0).all()), ".grad zeroed in place before the eager step"
    assert len(sg) == 0 and sg.fallbacks == 1, "graphs sized by the old reserve are dropped"
    log.clear()
    assert run("a", [p]) == ("graph", "a")
    assert log == [("capture", "a"), ("replay", "a")]
