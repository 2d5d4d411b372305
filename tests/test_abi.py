"""CPU: the C-ABI library loads and exports every symbol include/cvk.h declares (no compute calls)."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
    src = open(os.path.join(ROOT, "include", "cvk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cvk_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from cosyvoice_b200 import build, cvk
    build.build()
    lib = ctypes.CDLL(cvk.lib_path())
    names = _declared()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/cvk.h but not exported"
    assert set(names) == set(cvk.SIGNATURES), set(names) ^ set(cvk.SIGNATURES)


def test_create_fails_loudly_without_gpu():
    import torch
    from cosyvoice_b200 import cvk
    if torch.cuda.is_available():
        return
    lib = cvk.load_library()
    h = ctypes.c_void_p()
    assert lib.cvk_create(0, 1, 1 << 20, ctypes.byref(h)) != 0      # no CPU fallback
    try:
        cvk.Context()
    except RuntimeError as e:
        assert "no CPU fallback" in str(e)
    else:
        raise AssertionError("Context() must raise without a GPU")


def test_version_string():
    from cosyvoice_b200 import cvk
    assert b"sm_90a" in cvk.load_library().cvk_version()
