"""CPU tier: the C ABI.  The library must load without a GPU and export exactly the symbols include/macaw_b200.h
declares; the ctypes signature table must cover the same set.  No compute call is made here."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "macaw_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(mm_[a-z0-9_]+)\s*\(", src))


def test_header_library_and_ctypes_agree():
    from macaw_llm_b200 import _lib

    lib = _lib.load()  # builds with nvcc if missing
    syms = header_symbols()
    assert syms, "no symbols parsed from the header"
    assert syms == set(_lib.SIGNATURES), (syms ^ set(_lib.SIGNATURES))
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (mm_[a-z0-9_]+)", out))
    assert syms <= exported, syms - exported
    assert lib.mm_abi_version() == _lib.ABI_VERSION
    assert isinstance(lib.mm_launch_count(), int)


def test_struct_sizes_match_c_layout():
    """ctypes mirrors of mm_gemm_args / mm_attn_args must have the C layout (checked by compiling a probe)."""
    import ctypes
    import tempfile

    from macaw_llm_b200 import _lib

    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "macaw_b200.h"
int main(void){ printf("%zu %zu %zu %zu\n", sizeof(mm_gemm_args), offsetof(mm_gemm_args, rope_cols), sizeof(mm_attn_args), offsetof(mm_attn_args, scale)); return 0; }
'''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(probe)
        exe = os.path.join(d, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        a, b, c_, e = map(int, subprocess.run([exe], capture_output=True, text=True).stdout.split())
    assert ctypes.sizeof(_lib.GemmArgs) == a and _lib.GemmArgs.rope_cols.offset == b
    assert ctypes.sizeof(_lib.AttnArgs) == c_ and _lib.AttnArgs.scale.offset == e


def test_errors_are_reported_not_thrown():
    """Bad arguments come back as a non-zero code + message (no exception / abort crosses the ABI); validation
    happens before any CUDA call so this runs on a GPU-less box."""
    import ctypes

    from macaw_llm_b200 import _lib

    lib = _lib.load()
    rc = lib.mm_gemm_fwd(None, None)
    assert rc != 0 and b"null args" in lib.mm_last_error()
    a = _lib.GemmArgs()
    a.M, a.N, a.K, a.batch = 0, 8, 8, 1
    assert lib.mm_gemm_fwd(ctypes.byref(a), None) != 0 and b"bad shape" in lib.mm_last_error()
    assert lib.mm_rmsnorm_fwd(None, None, None, 1, 7, 1e-6, None) != 0


def test_integration_md_stub_matches_abi():
    """The ctypes stub shown to reference maintainers in INTEGRATION.md must mirror mm_gemm_args exactly."""
    import ctypes

    from macaw_llm_b200 import _lib

    src = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    block = src[src.index("class GemmArgs(C.Structure)"):src.index("def b200_linear")]
    ns = {}
    exec("import ctypes as C\n" + block, ns)
    doc = ns["GemmArgs"]
    assert [f[0] for f in doc._fields_] == [f[0] for f in _lib.GemmArgs._fields_]
    assert ctypes.sizeof(doc) == ctypes.sizeof(_lib.GemmArgs)


def test_product_kernels_are_hopper_native_sass():
    """Static check of the shipped cubin (cuobjdump, no GPU): the GEMM, flash-attention and fused alignment kernels carry
    wgmma (HGMMA) + TMA (UTMALDG) + mbarrier waits (SYNCS); no kernel in the library contains mma.sync (HMMA); nothing
    spills to local memory."""
    import shutil
    import sys

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from macaw_llm_b200 import _lib

    _lib.load()
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sass_inventory.py")], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = out.stdout.splitlines()
    hdr = next(l for l in lines if l.startswith("kernel "))
    cols = hdr.split()[1:]
    rows = {}
    for l in lines:
        if l.startswith(("#", "kernel ", "TOTAL")):
            continue
        m = re.match(r"(.+?)\s+((?:\d+\s+){%d}\d+)\s*$" % (len(cols) - 1), l)
        assert m, l
        rows[m.group(1).strip()] = dict(zip(cols, map(int, m.group(2).split())))
    for fam in ("gemm_bf16_kernel<", "fa_wgmma_kernel<", "align_fused_kernel"):
        fam_rows = {k: v for k, v in rows.items() if k.startswith(fam)}
        assert fam_rows, fam
        for k, v in fam_rows.items():
            assert v["HGMMA"] > 0 and v["UTMALDG"] > 0 and v["SYNCS"] > 0 and v["HMMA"] == 0, (k, v)
    assert not {k for k, v in rows.items() if v["HMMA"]}, {k: v["HMMA"] for k, v in rows.items() if v["HMMA"]}
    assert all(v["LOCAL"] == 0 for v in rows.values()), {k: v["LOCAL"] for k, v in rows.items() if v["LOCAL"]}
