"""The C-ABI shared library builds for sm_90a, loads without a GPU and exports every symbol include/dvla.h declares."""
import ctypes
import os
import re
import subprocess

import pytest

from dreamvla_b200 import _lib, build


@pytest.fixture(scope="module")
def lib_path():
    return build.build_library()


def declared_symbols(root):
    text = open(os.path.join(root, "include", "dvla.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dvla_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported(lib_path, repo_root):
    lib = ctypes.CDLL(lib_path)
    syms = declared_symbols(repo_root)
    assert len(syms) >= 19
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/dvla.h but not exported"
    assert sorted(_lib.EXPORTS) == syms, "dreamvla_b200/_lib.py EXPORTS out of sync with include/dvla.h"


def test_version_and_error_string(lib_path):
    lib = _lib.load()
    assert lib.dvla_version() == 100
    assert isinstance(lib.dvla_last_error(), bytes)


def test_invalid_args_return_error_not_abort(lib_path):
    lib = _lib.load()
    args = _lib.GemmArgs()           # all-null pointers
    rc = lib.dvla_gemm(ctypes.byref(args), None)
    assert rc == -1
    assert b"null" in lib.dvla_last_error()


def test_sass_is_hopper_native(lib_path):
    """wgmma / TMA / mbarrier transaction waits must be present in the SASS of the shipped library (HGMMA, UTMALDG, SYNCS)."""
    try:
        sass = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True, timeout=300).stdout
    except FileNotFoundError:
        pytest.skip("cuobjdump not available")
    assert "arch = sm_90a" in sass
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "UTMALDG", "SYNCS.PHASECHK.TRANS64"):
        assert mnemonic in sass, f"{mnemonic} missing from SASS"


def test_product_does_not_import_oracle(repo_root):
    bad = []
    for dp, _, files in os.walk(os.path.join(repo_root, "dreamvla_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "/root/reference" in src:
                    bad.append(os.path.join(dp, f))
    assert not bad, f"product path must not touch the oracle or the reference tree: {bad}"


def test_ops_fail_loudly_without_cuda():
    import torch
    from dreamvla_b200 import ops
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    w = torch.zeros(8, 64, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.linear(x, w)
