"""The C-ABI shared library builds for sm_90a, loads without a GPU and exports every symbol include/dvla.h declares; the
ctypes prototypes and Structures of dreamvla_b200/_lib.py match the header."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from dreamvla_b200 import _lib, build


@pytest.fixture(scope="module")
def lib_path():
    return build.build_library()


def header_text(root):
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "dvla.h")).read(), flags=re.S)


def declared_symbols(root):
    return sorted(set(re.findall(r"\b(dvla_[a-z0-9_]+)\s*\(", header_text(root))))


# C type of a dvla.h declaration -> the ctypes type _lib.PROTOTYPES must give it.  Every pointer is c_void_p, except the
# returned string of dvla_last_error.
C_TO_CTYPES = {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
               "float": ctypes.c_float}


def _ctype(decl, ret=False):
    t = re.sub(r"\s+", " ", decl).replace(" *", "*").strip()
    if ret and t == "const char*":
        return ctypes.c_char_p
    if "*" in t:
        return ctypes.c_void_p
    return C_TO_CTYPES[t.replace("const ", "")]


def header_prototypes(root):
    """name -> (restype, [argtypes]) of every function include/dvla.h declares."""
    protos = {}
    for decl in header_text(root).split(";"):
        m = re.search(r"([A-Za-z_][\w\s*]*?)\b(dvla_\w+)\s*\(([^()]*)\)\s*$", decl)
        if not m:
            continue
        ret, name, params = m.groups()
        params = [p.strip() for p in params.split(",")]
        argtypes = [] if params == ["void"] else [_ctype(re.fullmatch(r"(.*?)\s*\w+", p).group(1)) for p in params]
        protos[name] = (_ctype(ret, ret=True), argtypes)
    return protos


def prototype_mismatches(table, header):
    bad = [f"{n}: declared in dvla.h, missing from the table" for n in sorted(set(header) - set(table))]
    bad += [f"{n}: in the table, not declared in dvla.h" for n in sorted(set(table) - set(header))]
    for n in sorted(set(table) & set(header)):
        restype, argtypes = table[n]
        if restype is not header[n][0] or list(argtypes) != header[n][1]:
            bad.append(f"{n}: table {restype.__name__}({', '.join(t.__name__ for t in argtypes)}), dvla.h "
                       f"{header[n][0].__name__}({', '.join(t.__name__ for t in header[n][1])})")
    return bad


# every ctypes mirror of a dvla.h struct
STRUCTS = {_lib.GemmArgs: "dvla_gemm_args", _lib.GemmPlanInfo: "dvla_gemm_plan_info",
           _lib.LayerNormFwdArgs: "dvla_layernorm_fwd_args", _lib.LayerNormBwdArgs: "dvla_layernorm_bwd_args",
           _lib.AttnFwdArgs: "dvla_attn_fwd_args", _lib.AttnBwdArgs: "dvla_attn_bwd_args", _lib.AdamWArgs: "dvla_adamw_args",
           _lib.AdamWMasterArgs: "dvla_adamw_master_args", _lib.ImageFnArgs: "dvla_image_fn_args",
           _lib.DitBlockWeights: "dvla_dit_block_weights", _lib.DitSamplerArgs: "dvla_dit_sampler_args"}


@pytest.fixture(scope="module")
def c_layout(repo_root, tmp_path_factory):
    """(struct, field) -> (offset, size) and (struct, None) -> (0, sizeof) of the STRUCTS fields, as the host C compiler (the
    one nvcc builds the library's host code with) lays out include/dvla.h."""
    cc = shutil.which(os.environ.get("CC", "cc")) or shutil.which("gcc")
    assert cc, "no host C compiler found (building the library needs one too)"
    src = ["#include <stddef.h>", "#include <stdio.h>", '#include "dvla.h"', "int main(void) {"]
    for cls, cname in STRUCTS.items():
        src.append(f'  printf("{cname} - 0 %zu\\n", sizeof({cname}));')
        for field, *_ in cls._fields_:
            src.append(f'  printf("{cname} {field} %zu %zu\\n", offsetof({cname}, {field}), sizeof((({cname}*)0)->{field}));')
    src.append("  return 0;\n}\n")
    d = tmp_path_factory.mktemp("layout")
    (d / "layout.c").write_text("\n".join(src))
    subprocess.run([cc, "-I", os.path.join(repo_root, "include"), "-o", str(d / "layout"), str(d / "layout.c")], check=True)
    out = subprocess.run([str(d / "layout")], capture_output=True, text=True, check=True).stdout
    layout = {}
    for line in out.splitlines():
        cname, field, offset, size = line.split()
        layout[(cname, None if field == "-" else field)] = (int(offset), int(size))
    return layout


def struct_mismatches(cls, cname, layout):
    bad = []
    if ctypes.sizeof(cls) != layout[(cname, None)][1]:
        bad.append(f"sizeof({cname}) = {layout[(cname, None)][1]}, {cls.__name__}: {ctypes.sizeof(cls)}")
    for field, *_ in cls._fields_:
        d = getattr(cls, field)
        if (d.offset, d.size) != layout[(cname, field)]:
            bad.append(f"{cname}.{field} at {layout[(cname, field)]} (offset, size), {cls.__name__}: {(d.offset, d.size)}")
    return bad


def test_header_symbols_exported(lib_path, repo_root):
    lib = ctypes.CDLL(lib_path)
    syms = declared_symbols(repo_root)
    assert len(syms) >= 19
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/dvla.h but not exported"
    assert sorted(_lib.EXPORTS) == syms, "dreamvla_b200/_lib.py EXPORTS out of sync with include/dvla.h"


def test_prototypes_match_header(repo_root):
    assert prototype_mismatches(_lib.PROTOTYPES, header_prototypes(repo_root)) == []


@pytest.mark.parametrize("cls", list(STRUCTS), ids=lambda c: c.__name__)
def test_structs_match_header(c_layout, cls):
    assert struct_mismatches(cls, STRUCTS[cls], c_layout) == []


def test_abi_checks_catch_mutations(c_layout, repo_root):
    fields = list(_lib.GemmArgs._fields_)
    names = [f[0] for f in fields]
    i, j = names.index("M"), names.index("N")
    fields[i], fields[j] = fields[j], fields[i]
    swapped = type("GemmArgs", (ctypes.Structure,), {"_fields_": fields})
    assert struct_mismatches(swapped, "dvla_gemm_args", c_layout)
    truncated = type("AdamWArgs", (ctypes.Structure,), {"_fields_": _lib.AdamWArgs._fields_[:-1]})
    assert struct_mismatches(truncated, "dvla_adamw_args", c_layout)
    table = dict(_lib.PROTOTYPES)
    restype, argtypes = table["dvla_colsum_accum"]
    table["dvla_colsum_accum"] = (restype, [argtypes[0], ctypes.c_int, *argtypes[2:]])    # int64_t rows as C int
    assert prototype_mismatches(table, header_prototypes(repo_root))


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
