"""The C-ABI library loads and exports every symbol include/esvit_b200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

from esvit_b200 import _lib, build


def _header_decls():
    src = open(_lib.HEADER_PATH).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    decls = {}
    for m in re.finditer(r"\bint\s+(esvit_\w+)\s*\(([^)]*)\)\s*;", src):
        args = m.group(2).strip()
        n = 0 if args in ("", "void") else len(args.split(","))
        decls[m.group(1)] = n
    return decls


def test_library_builds_and_exports_every_declared_symbol():
    path = build.build()
    assert os.path.isfile(path)
    lib = ctypes.CDLL(path)
    decls = _header_decls()
    assert len(decls) >= 25
    for name in decls:
        assert hasattr(lib, name), f"{name} declared in include/esvit_b200.h but not exported"


def test_ctypes_signatures_match_header():
    decls = _header_decls()
    assert set(decls) == set(_lib.SIGNATURES), set(decls) ^ set(_lib.SIGNATURES)
    for name, n in decls.items():
        assert len(_lib.SIGNATURES[name]) == n, name


def test_no_cpu_fallback_when_library_missing(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libesvit_b200.so")
    with pytest.raises(_lib.EsvitKernelError):
        _lib.load()


def test_sass_is_sm90a():
    out = os.popen(f"cuobjdump -lelf {build.LIB} 2>/dev/null").read()
    if not out:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out
