"""The C-ABI library loads and exports every symbol include/b2v.h declares (CPU-only:
no compute call is made)."""
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def header_symbols():
    txt = (ROOT / "include" / "b2v.h").read_text()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(b2v_[a-z0-9_]+)\s*\(", txt)))


def test_library_builds_and_exports_header_symbols():
    from invesalius3_b200 import _build, _lib
    _build.build_cuda()
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(lib, s), f"libb2v.so does not export {s}"
    assert sorted(_lib.PROTOTYPES) == syms, "ctypes prototypes and include/b2v.h disagree"
    assert lib.b2v_version() >= 100
    assert lib.b2v_last_error() is not None


def test_sass_is_sm90a():
    import subprocess
    from invesalius3_b200 import _build
    lib = _build.build_cuda()
    out = subprocess.run(["cuobjdump", "-lelf", str(lib)], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_product_does_not_import_oracle():
    """The product path must never route through the CPU oracle."""
    for p in (ROOT / "invesalius3_b200").rglob("*.py"):
        src = p.read_text()
        assert not re.search(r"^\s*(import|from)\s+oracle\b", src, flags=re.M), f"{p} imports the oracle"
    for p in (ROOT / "invesalius3_b200" / "csrc").glob("*"):
        if p.is_file() and p.suffix in (".cu", ".cuh", ".h"):
            assert "oracle" not in p.read_text().lower() or p.name == "mc_tables.h", p


def test_header_is_plain_c_and_a_c_program_links(tmp_path):
    """include/b2v.h is the boundary for compiled callers: it must be valid C99 and C++11 on its own,
    and a C program must link against libb2v.so with nothing else (no torch, no Python)."""
    import subprocess
    from invesalius3_b200 import _build
    lib = _build.build_cuda()
    src = tmp_path / "caller.c"
    src.write_text('#include <stdio.h>\n#include "b2v.h"\n'
                   "int main(void) {\n"
                   "  /* addresses only: no device work on a box without a GPU */\n"
                   "  void* fns[] = {(void*)b2v_threshold_i16, (void*)b2v_floodfill_threshold, (void*)b2v_mc_count,\n"
                   "                 (void*)b2v_mc_emit, (void*)b2v_mida, (void*)b2v_ws_flood};\n"
                   '  printf("%d %d\\n", b2v_version(), (int)(sizeof fns / sizeof fns[0]));\n'
                   "  return 0;\n}\n")
    inc = str(ROOT / "include")
    for cc, std, name in (("gcc", "-std=c99", "caller.c"), ("g++", "-std=c++11", "caller.cpp")):
        f = tmp_path / name
        f.write_text(src.read_text())
        r = subprocess.run([cc, std, "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", inc, str(f)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    exe = tmp_path / "caller"
    r = subprocess.run(["gcc", "-std=c99", "-I", inc, str(src), "-o", str(exe), str(lib),
                        f"-Wl,-rpath,{lib.parent}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.split() == [str(_lib_version()), "6"], (out.stdout, out.stderr)


def _lib_version():
    from invesalius3_b200 import _lib
    return _lib.load().b2v_version()
