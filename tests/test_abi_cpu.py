"""CPU tests of the C-ABI boundary: the library loads, exports every symbol include/h2b200.h declares, fails loudly
without a GPU (no CPU fallback), and keeps errors on the right side of the boundary.  No compute calls."""
import ctypes as C
import os
import re
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    import halo2_lib_b200 as h
    syms = h.header_symbols()
    assert len(syms) >= 35
    raw = C.CDLL(h.LIB_PATH)
    for s in syms:
        assert hasattr(raw, s), f"{s} declared in include/h2b200.h but not exported by libh2b200.so"
        assert s in h.SIGNATURES, f"{s} has no ctypes signature"
    h.lib.h2b_version.restype = C.c_char_p
    assert b"h2b200" in h.lib.h2b_version() and b"sm_90a" in h.lib.h2b_version()


def test_no_cpu_fallback_without_gpu():
    import torch
    import halo2_lib_b200 as h
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(h.H2BError) as ei:
        h.Context(0)
    assert ei.value.code == -2 and "no CPU fallback" in str(ei.value)
    # null-context calls report H2B_ERR_ARG instead of crashing
    assert h.lib.h2b_ctx_synchronize(None) == -1
    assert h.lib.h2b_msm_g1(None, None, 0, None, 0, None) == -1


def test_domain_constants_match_oracle():
    import halo2_lib_b200 as h
    from oracle import oracle as orc, pyref
    from util import unmont
    for k in (0, 1, 5, 19, 21, 28):
        w = h.omega(k)
        assert np.array_equal(w, orc.omega(k))
        assert unmont(w.reshape(1, 4), pyref.R) == [pyref.omega_for(k)]
    with pytest.raises(h.H2BError):
        h.omega(29)


def test_product_does_not_reference_the_oracle():
    """The shipped path (package + csrc + C++ mirror) must not import, link or call anything under oracle/."""
    bad = []
    for base in ("halo2-lib_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".inc", "Makefile")):
                    txt = open(os.path.join(dirpath, f), errors="ignore").read()
                    if re.search(r"(import\s+oracle|from\s+oracle|liboracle|orc_[a-z_]+\s*\()", txt):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_bench_schedule_shape():
    import bench
    s = bench.Schedule(3)
    assert len(s.msm) == 12  # SURVEY.md §8: 12 MSMs x 2^19 for the ECDSA circuit
    assert sorted(j for p in s.phases for j in p) == list(range(12))
    a = bench.witness_like(np.random.default_rng(0), 4096)
    frac0 = float((a == 0).all(axis=1).mean())
    assert 0.30 < frac0 < 0.40


def test_graph_struct_layout_matches_the_header(tmp_path):
    """the ctypes twin of h2b_graph (and with it the oracle's orc_graph, which tests fill through the same structure) has
    the size and field offsets the C compiler gives the header's struct"""
    import ctypes as C
    import subprocess
    from halo2_lib_b200._capi import Graph, HEADER_PATH
    fields = [f[0] for f in Graph._fields_]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void) {\n  printf("%%zu", sizeof(h2b_graph));\n%s  return 0;\n}\n'
                   % (HEADER_PATH, "".join('  printf(" %%zu", offsetof(h2b_graph, %s));\n' % f for f in fields)))
    exe = tmp_path / "layout"
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.check_call([cc, "-std=c11", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(Graph)
    assert got[1:] == [getattr(Graph, f).offset for f in fields]


def test_rust_ffi_declares_every_header_symbol():
    """rust/halo2-b200/src/ffi.rs is generated from include/h2b200.h (tools/gen_rust_ffi.py): it must be up to date, declare
    every exported function exactly once, and agree with the ctypes table on the number of arguments (no Rust toolchain
    exists in this image, so this is the structural check)."""
    import subprocess, sys
    from halo2_lib_b200._capi import SIGNATURES, header_symbols
    path = os.path.join(ROOT, "rust", "halo2-b200", "src", "ffi.rs")
    before = open(path).read()
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_rust_ffi.py")], stdout=subprocess.DEVNULL)
    assert open(path).read() == before, "ffi.rs is stale: run tools/gen_rust_ffi.py"
    decl = dict(re.findall(r"pub fn (h2b_[a-z0-9_]+)\(([^)]*)\)", before))
    assert sorted(decl) == header_symbols()
    for name, args in decl.items():
        n_args = 0 if not args.strip() else len(args.split(","))
        assert n_args == len(SIGNATURES[name][1]), name
    for f in ("Cargo.toml", "build.rs", "src/lib.rs", "src/backend.rs"):
        assert os.path.exists(os.path.join(ROOT, "rust", "halo2-b200", f))
    # every ffi function the safe wrappers call is declared
    used = set(re.findall(r"\b(h2b_[a-z0-9_]+)\(", open(os.path.join(ROOT, "rust", "halo2-b200", "src", "backend.rs")).read()))
    assert used <= set(decl), used - set(decl)
