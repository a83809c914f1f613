"""CPU checks of the drop-in boundary: the C-ABI library builds, loads, and exports every symbol that
include/sdetr_b200.h declares; the ctypes signature table covers exactly that set.  (No compute calls here --
there is no GPU in the build container; the parity tests proper are tests/test_gpu_parity.py, -m gpu.)"""
import ctypes
import os
import re

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "sdetr_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sdetr_[a-z0-9_]+)\s*\(", text)))


@pytest.fixture(scope="module")
def pkg():
    import __graft_entry__ as entry
    entry.build()
    import salience_detr_b200 as p
    return p


def test_header_declares_the_path():
    syms = declared_symbols()
    for must in ("sdetr_msda_forward", "sdetr_msda_backward", "sdetr_msda_fused_forward", "sdetr_salience_select",
                 "sdetr_token_gather", "sdetr_token_scatter", "sdetr_background_embed"):
        assert must in syms


def test_library_exports_every_declared_symbol(pkg):
    cdll = ctypes.CDLL(pkg.cabi.LIB_PATH)
    for s in declared_symbols():
        assert hasattr(cdll, s), f"{s} declared in include/sdetr_b200.h but not exported"


def test_ctypes_table_matches_header(pkg):
    assert sorted(pkg.cabi.SIGNATURES) == declared_symbols()
    # argument counts of the table == the header's parameter lists
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    for name, (_, args) in pkg.cabi.SIGNATURES.items():
        m = re.search(r"\b%s\s*\(([^;]*?)\)\s*;" % name, text, flags=re.S)
        assert m, name
        params = m.group(1).strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(args), f"{name}: header has {n} parameters, ctypes table {len(args)}"


def test_library_is_sm90a_and_torch_free(pkg):
    import subprocess
    out = subprocess.run(["cuobjdump", "--list-elf", pkg.cabi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    ldd = subprocess.run(["ldd", pkg.cabi.LIB_PATH], capture_output=True, text=True).stdout
    # plain C-ABI: no torch types behind the boundary.  The names and resolved paths are checked, without the load
    # addresses ldd prints: those are random and may contain "c10" as hex digits
    deps = re.sub(r"\(0x[0-9a-fA-F]+\)", "", ldd)
    assert "libc.so" in deps and "torch" not in deps and "c10" not in deps, deps


def test_version_and_error_string(pkg):
    lib = pkg.cabi.lib()
    assert lib.sdetr_version() >= 100
    assert isinstance(lib.sdetr_last_error(), bytes)
    # argument validation happens before any CUDA call, so it is testable without a GPU
    rc = lib.sdetr_topk_desc(None, 1, 10, 3, None, None, 0, None)
    assert rc == -1 and b"null pointer" in lib.sdetr_last_error()
    assert lib.sdetr_salience_select_workspace(2, 22323, 4) >= 8 * 2 * 22323 * 4


def test_product_path_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under salience-detr_b200/ may reference it."""
    pkgdir = os.path.join(ROOT, "salience-detr_b200")
    for dirpath, _, files in os.walk(pkgdir):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("the oracle (torch leaves it unspecified)", "").replace(
                    "shared with the oracle", ""), os.path.join(dirpath, f)


def test_argument_validation_of_the_later_entry_points(pkg):
    """Shape / bound checks run on the host before any CUDA call, so they are testable without a GPU."""
    lib = pkg.cabi.lib()
    buf = (ctypes.c_float * 1024)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    # a feature map larger than the learned embedding tables is an index error in the reference (nn.Embedding)
    shapes = (ctypes.c_int64 * 4)(4, 12, 2, 6)
    rc = lib.sdetr_background_embed(p, p, p, 1, 1, p, p, 8, p, ctypes.cast(shapes, ctypes.c_void_p), p, 1, 60, 64, 2, p, None)
    assert rc == -1 and b"embedding tables hold 8" in lib.sdetr_last_error()
    # the fused pre-attention kernels are specialised for the reference's width
    rc = lib.sdetr_mha_in_proj(p, p, p, 1, 10, 5, 128, p, p, p, p, None)
    assert rc != 0 and b"only 256" in lib.sdetr_last_error()
    rc = lib.sdetr_mha_out_proj_ln_scatter(p, p, p, p, p, p, 1e-5, p, p, p, None, 1, 10, 5, 256, None)
    assert rc == -1 and b"go together" in lib.sdetr_last_error()
    rc = lib.sdetr_attention_qkv(p, p, 1, 10, 2, 64, None)
    assert rc != 0 and b"head_dim 64" in lib.sdetr_last_error()
    rc = lib.sdetr_gelu_colmean(p, 1, 10, 30, 16, p, 1 << 20, None)
    assert rc == -1 and b"bad sizes" in lib.sdetr_last_error()
    assert lib.sdetr_gelu_colmean_workspace(2, 16800, 256, 128) >= 2 * 296 * 128 * 4
    rc = lib.sdetr_gemm_3xtf32_pre(p, 40, p, p, None, p, 8, 4, 8, 40, 0, None)
    assert rc != 0 and b"multiple of 32" in lib.sdetr_last_error()
    assert lib.sdetr_ffn_fused_workspace_floats(1000, 2048) == 1000 * (2048 + 256)
    assert lib.sdetr_ffn_fused_workspace_floats(1000, 2000) == 0  # hidden width must be a multiple of 128
