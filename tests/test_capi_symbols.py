"""CPU-only: the C-ABI library loads and exports every symbol include/fg_b200.h declares (no compute)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "fg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fg_[a-zA-Z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from face_generator_b200.lib import SYMBOLS, load_library
    lib = load_library()
    names = header_symbols()
    assert len(names) >= 45
    for n in names:
        assert hasattr(lib, n), "libfg_b200.so does not export %s" % n
    assert sorted(SYMBOLS) == names, "python binding and header disagree: %s" % (set(SYMBOLS) ^ set(names))
    assert b"sm_90a" in lib.fg_version()


def test_no_cpu_fallback_create_fails_loudly_without_gpu():
    import face_generator_b200 as fg
    import ctypes
    try:
        ctypes.CDLL("libcuda.so.1")
        has_driver = True
    except OSError:
        has_driver = False
    if has_driver:
        pytest.skip("a CUDA driver is present; this check is for the CPU-only container")
    with pytest.raises(fg.FGError):
        fg.Context(0, 8, 3)


def test_hyper_defaults_match_train_lua():
    import face_generator_b200 as fg
    h = fg.hyper_default()
    # train.lua:16-50 and interruptable_optimizers.lua:53-57
    assert abs(h.lr_D - 1e-3) < 1e-9 and abs(h.lr_G - 1e-3) < 1e-9
    assert abs(h.beta1 - 0.9) < 1e-7 and abs(h.beta2 - 0.999) < 1e-7 and abs(h.eps - 1e-8) < 1e-12
    assert h.D_L1 == 0 and abs(h.D_L2 - 1e-4) < 1e-9 and h.G_L1 == 0 and h.G_L2 == 0
    assert h.D_clamp == 1 and h.G_clamp == 5 and abs(h.D_maxAcc - 1.01) < 1e-6
    assert abs(h.p_spatial - 0.2) < 1e-7 and abs(h.p_drop - 0.5) < 1e-7


def test_param_counts_match_reference_models():
    from face_generator_b200.lib import load_library
    from oracle import oracle as O
    lib = load_library()
    for C in (1, 3):
        assert lib.fg_param_count(0, C) == O.G_param_count(C)
        assert lib.fg_param_count(1, C) == O.D_param_count(C)
    assert lib.fg_param_count(0, 3) == 2470406  # SURVEY.md 8a
    assert lib.fg_param_count(1, 3) == 2863239  # 2 863 233 w+b + 6 PReLU slopes (models.lua:382-416)


def test_lua_ffi_cdef_declares_every_symbol():
    """face_generator_b200/lua/fg_ffi.lua (the binding a Torch maintainer loads) must cdef the whole header."""
    lua = open(os.path.join(ROOT, "face_generator_b200", "lua", "fg_ffi.lua")).read()
    declared = set(re.findall(r"\b(fg_[a-zA-Z0-9_]+)\s*\(", lua))
    missing = [n for n in header_symbols() if n not in declared]
    assert not missing, missing


def test_lua_shims_only_call_declared_entry_points():
    """Every C.fg_* / C['fg_*'] the Lua shims reference exists in include/fg_b200.h (LuaJIT cannot run here, so at
    least the names are checked)."""
    names = set(header_symbols())
    lua_dir = os.path.join(ROOT, "face_generator_b200", "lua")
    used = set()
    for fn in os.listdir(lua_dir):
        src = open(os.path.join(lua_dir, fn)).read()
        if fn != "fg_ffi.lua":
            used |= set(re.findall(r"C\.(fg_[a-zA-Z0-9_]+)", src))
            used |= set(re.findall(r"'(fg_[a-z0-9_]+_(?:forward|backward))'", src))
    assert used and not (used - names), sorted(used - names)
