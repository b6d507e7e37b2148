"""Every C checker is built into the one oracle library, oracle/liboracle.so, by one make call, and every
checker module loads it through the package's single loader (CPU-only)."""
import ctypes as C
import importlib
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
ORACLE = ROOT / "oracle"


def called_symbols():
    """The orc_* names oracle/*.py calls through lib(): lib().orc_x, and getattr(lib(), f"orc_x_{suf}") for
    every dtype suffix of the package."""
    import oracle
    names = set()
    for p in ORACLE.glob("*.py"):
        src = p.read_text()
        names.update(re.findall(r"\blib\(\)\.(orc_[a-z0-9_]+)", src))
        for stem in re.findall(r"getattr\(lib\(\), f\"(orc_[a-z0-9_]+)\{suf\}\"\)", src):
            names.update(stem + suf for suf in oracle._SUFFIX.values())
    return sorted(names)


def checker_modules():
    return sorted(p.stem for p in ORACLE.glob("*.py") if p.stem != "__init__" and "lib()" in p.read_text())


def test_library_exports_every_called_symbol():
    from invesalius3_b200 import _build
    so = _build.build_oracle()
    assert so == ORACLE / "liboracle.so"
    lib = C.CDLL(str(so))
    syms = called_symbols()
    assert len(syms) >= 45
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"liboracle.so does not export {missing}"


@pytest.mark.parametrize("name", checker_modules())
def test_checker_loads_the_one_library(name):
    import oracle
    mod = importlib.import_module(f"oracle.{name}")
    assert mod.lib() is oracle.lib()


@pytest.mark.parametrize("force", [False, True])
def test_build_oracle_runs_make_once(monkeypatch, force):
    from invesalius3_b200 import _build
    calls = []

    def run(cmd, **kw):
        calls.append(list(cmd))
        return subprocess.CompletedProcess(cmd, 0, "", "")

    monkeypatch.setattr(subprocess, "run", run)
    assert _build.build_oracle(force=force) == ORACLE / "liboracle.so"
    assert calls == [["make", "-C", str(ORACLE), *(["-B"] if force else [])]]
