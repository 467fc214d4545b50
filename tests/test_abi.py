"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every
symbol include/b200dqn.h declares (no compute calls — there is no GPU here), and the product
never imports the oracle."""
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    from simple_dqn_b200 import _lib as L
    if shutil.which("nvcc"):
        from simple_dqn_b200.build import build
        build()
    return L.load()


def header_symbols():
    text = open(os.path.join(ROOT, "include", "b200dqn.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200dqn_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol(lib):
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(lib, s), "libb200dqn.so does not export %s" % s
    out = subprocess.check_output(["nm", "-D", "--defined-only", lib._name], text=True)
    exported = set(re.findall(r" T (b200dqn_[a-z0-9_]+)", out))
    assert set(syms) <= exported
    # and the ctypes table binds exactly the declared set
    from simple_dqn_b200 import _lib as L
    assert set(L.EXPORTS) == set(syms)


def test_version_and_error_channel(lib):
    assert lib.b200dqn_version() == 100
    assert isinstance(lib.b200dqn_last_error(), bytes)


def test_config_default_matches_reference_flags(lib):
    import ctypes as C
    from simple_dqn_b200 import _lib as L
    cfg = L.NetConfig()
    assert lib.b200dqn_net_config_default(C.byref(cfg), 4) == 0
    # /root/reference/src/main.py:27-63 defaults
    assert (cfg.batch_size, cfg.history_length, cfg.screen_h, cfg.screen_w) == (32, 4, 84, 84)
    assert (cfg.discount_rate, cfg.learning_rate, cfg.decay_rate, cfg.clip_error) == (0.99, 0.00025, 0.95, 1.0)
    assert (cfg.min_reward, cfg.max_reward, cfg.target_steps) == (-1, 1, 10000)
    # the reward bounds are floats (main.py:43-44): a fractional bound crosses the boundary unchanged
    fields = dict(L.NetConfig._fields_)
    assert fields["min_reward"] is C.c_double and fields["max_reward"] is C.c_double
    assert "double min_reward;" in open(os.path.join(ROOT, "include", "b200dqn.h")).read()


def test_binary_is_hopper_native():
    """The shipped cubin targets sm_90a (and nothing else), the GEMM-shaped kernels run on warpgroup MMAs, conv1
    loads its frames from the ring inside its warpgroup-MMA kernel and fetches its weight tiles by TMA bulk copy, and
    the replay gather uses the TMA bulk-copy engine."""
    from simple_dqn_b200.build import NVCC
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from simple_dqn_b200 import _lib as L
    elf = subprocess.check_output([cuobjdump, "-lelf", L.LIB_PATH], text=True)
    archs = set(re.findall(r"\.(sm_\w+)\.cubin", elf))
    assert archs == {"sm_90a"}, archs
    sass = subprocess.check_output([cuobjdump, "-sass", L.LIB_PATH], text=True, stderr=subprocess.STDOUT)
    for shape in ("64x32x16", "64x64x16", "64x128x16"):
        assert "HGMMA.%s.F32" % shape in sass, shape
    conv1 = sass[sass.index("k_umma2INS_10V2Conv1FwdILi4E"):]
    conv1 = conv1[:conv1.index("Function :")] if "Function :" in conv1 else conv1
    for op in ("HGMMA.64x64x16.F32", "LDG.E", "UBLKCP"):
        assert op in conv1, op
    gather = sass[sass.index("k_gather"):]
    gather = gather[:gather.index(".....", 200) if "....." in gather[200:] else len(gather)]
    assert "UBLKCP" in gather


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "simple_dqn_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "oracle/" not in src or f.endswith((".cu", ".cuh")), f


def test_missing_library_fails_loudly(monkeypatch):
    from simple_dqn_b200 import _lib as L
    monkeypatch.setattr(L, "_lib", None)
    monkeypatch.setattr(L, "LIB_PATH", "/nonexistent/libb200dqn.so")
    with pytest.raises(ImportError, match="no CPU fallback"):
        L.load()


def test_argument_errors_surface_before_any_device_work():
    """Argument validation of the C-ABI happens ahead of the first CUDA call, so it can be exercised without a GPU:
    a ring smaller than the 8-frame ingestion bank (ADVICE r1: the deferred flush may wrap at most once) and an
    unknown optimizer / math mode are EINVAL -> AssertionError, the reference's error convention."""
    import ctypes as C

    import pytest

    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    with pytest.raises(AssertionError):
        L.call("b200dqn_replay_create", 0, 4, 84, 84, 4, 32, C.byref(h))
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.optimizer == L.OPT_RMSPROP and cfg.batch_size == 32
    cfg.optimizer = 7
    with pytest.raises(AssertionError):
        L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
