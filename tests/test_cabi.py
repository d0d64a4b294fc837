"""The C-ABI library builds, loads, and exports every symbol include/patchmatch_b200.h declares.
No compute is issued (argument validation returns before any CUDA call), so this runs without a GPU."""
import ctypes
import os
import re

import pytest

from patchmatchnet_b200 import _native

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(REPO, "include", "patchmatch_b200.h")


@pytest.fixture(scope="module")
def lib():
    _native.build_library()  # no-op when libpmb200.so is newer than its sources
    return _native.lib()


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(pmb200_[a-z_0-9]+)\s*\(", text)))


def test_header_symbols_are_all_exported(lib):
    names = declared_symbols()
    assert len(names) >= 12
    raw = ctypes.CDLL(_native.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
    assert set(names) == set(_native.EXPORTED_SYMBOLS), "ctypes binding and header disagree"


def declared_parameter_counts():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    counts = {}
    for name, params in re.findall(r"\b(pmb200_[a-z_0-9]+)\s*\(([^;{}]*?)\)\s*;", text, flags=re.S):
        params = params.strip()
        counts[name] = 0 if params in ("", "void") else params.count(",") + 1
    return counts


def test_ctypes_signatures_have_the_headers_parameter_counts():
    """A binding with one argument too many only fails when the entry point is first CALLED -- on the GPU box (round 2, run
    3 lost a GPU call to exactly that).  The declaration in the header is the contract: same number of parameters."""
    counts = declared_parameter_counts()
    assert set(counts) == set(_native._SIGNATURES)
    for name, (_res, args) in _native._SIGNATURES.items():
        assert len(args) == counts[name], f"{name}: ctypes binding has {len(args)} parameters, the header declares {counts[name]}"


def test_library_is_sm90a_only():
    import subprocess

    out = subprocess.run(["cuobjdump", "--list-elf", _native.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert not re.search(r"sm_(?!90a)\d+", out), out


def test_abi_version_and_errors_without_gpu(lib):
    assert lib.pmb200_abi_version() == 1
    # null pointers / bad sizes are rejected with PMB200_EINVAL before anything touches CUDA
    assert lib.pmb200_warp_corr(None, None, None, None, None, None, 1, 1, 16, 4, 4, 4, 4, 4, 1, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    assert lib.pmb200_warp_corr(one, one, one, one, None, one, 1, 1, 16, 5, 4, 4, 4, 4, 1, None) == -1
    assert lib.pmb200_warp_corr(one, one, one, one, None, one, 99, 1, 16, 4, 4, 4, 4, 4, 1, None) == -1
    # neighbour counts the reference raises NotImplementedError for -> PMB200_EUNSUPPORTED
    assert lib.pmb200_offset_corr(one, one, 0, one, 1, 16, 4, 4, 4, 10, 2, None) == -2
    assert lib.pmb200_init_propagate(one, one, 0, one, one, one, None, 1, 1, 1, 4, 4, 8, 5, 2, 0.1, None) == -2
    assert lib.pmb200_adaptive_eval(one, one, None, None, one, 0, one, one, one, one, one, 1, 8, 4, 4, 11, 2, 0.1, 0, None) == -2
    assert lib.pmb200_init_propagate(one, one, 0, one, one, one, None, 1, 0, 1, 4, 4, 16, 8, 2, 0.1, None) == -1  # random init has 48


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_native, "LIB_PATH", str(tmp_path / "nope.so"))
    monkeypatch.setattr(_native, "_lib", None)
    with pytest.raises(_native.NativeLibraryMissing):
        _native.lib()
