"""The C-ABI shared library builds for sm_90a, loads without a GPU and exports every symbol include/cvvae_b200.h
declares (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "cvvae_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cvvae_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported():
    import __graft_entry__ as ge
    ge.build()
    from cvvae_b200 import _lib
    lib = ctypes.CDLL(_lib.LIBPATH)
    names = _declared()
    assert len(names) >= 18, names
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/cvvae_b200.h but not exported"
    # the ctypes binding covers the same set
    assert set(names) == set(_lib.EXPORTS), set(names) ^ set(_lib.EXPORTS)
    assert lib.cvvae_abi_version() == _lib.ABI_VERSION


def test_struct_layouts_match_header():
    from cvvae_b200 import _lib
    # cvvae_tensor5: pointer + 5 x int32 (+4 pad) + 5 x int64
    assert ctypes.sizeof(_lib.Tensor5) == 8 + 5 * 4 + 4 + 5 * 8
    d = _lib.ConvDesc()
    assert _lib.ConvDesc.gn_groups.offset > _lib.ConvDesc.gn_stats.offset > _lib.ConvDesc.alpha.offset
    assert ctypes.sizeof(d) % 8 == 0


def test_no_cpu_fallback_without_library(monkeypatch, tmp_path):
    from cvvae_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIBPATH", str(tmp_path / "missing.so"))
    import pytest
    with pytest.raises(_lib.CvvaeError, match="missing"):
        _lib.load()
