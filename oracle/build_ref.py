"""Build the REAL reference kernels into ``oracle/_ref/`` (test infrastructure only).

Compiles the reference's own Cython sources *where they lie* in a moleculekit source checkout named by the
environment variable ``MKB_REFERENCE_SRC`` (``moleculekit/occupancy_utils/occupancy_utils.pyx`` and
``moleculekit/distance_utils/distance_utils.pyx``) with the reference's own flags
(``setup.py:41-53``: ``language="c++"``, ``-O3``, numpy include, Py_LIMITED_API 0x030B0000).
Nothing is copied into the repository: the generated C++ goes to a temp dir that is
deleted, and only the ``.so`` files land in ``oracle/_ref/`` (git-ignored).  Without a checkout the tests that
compare with these binaries skip; the stored fixtures under tests/golden/ carry their outputs.

We do NOT run the reference's build system (setup.py); this is a three-command recipe:
``cython --cplus`` -> ``g++ -O3 -shared -fPIC``.

Usage:  python oracle/build_ref.py [--reference <moleculekit checkout>] [--force]
"""
from __future__ import annotations

import argparse
import os
import shutil
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

MODULES = {
    "occupancy_utils": "moleculekit/occupancy_utils/occupancy_utils.pyx",
    "distance_utils": "moleculekit/distance_utils/distance_utils.pyx",
    "bondguesser_utils": "moleculekit/bondguesser_utils/bondguesser_utils.pyx",
    "wrapping": "moleculekit/wrapping/wrapping.pyx",
    "atomselect_utils": "moleculekit/atomselect_utils/atomselect_utils.pyx",
    "xtc": "moleculekit/fileformats/xtc/xtc.pyx",
    "hbonds": "moleculekit/interactions/hbonds/hbonds.pyx",
    "pipi": "moleculekit/interactions/pipi/pipi.pyx",
    "cationpi": "moleculekit/interactions/cationpi/cationpi.pyx",
    "sigmahole": "moleculekit/interactions/sigmahole/sigmahole.pyx",
}

# extra C++ sources / include directories of a module (the reference's setup.py:55-66 lists the same files)
EXTRA_SOURCES = {
    "xtc": ["moleculekit/fileformats/xtc/src/xdrfile_xtc.cpp", "moleculekit/fileformats/xtc/src/xdrfile.cpp",
            "moleculekit/fileformats/xtc/src/xtc_src.cpp"],
}
EXTRA_INCLUDES = {
    "xtc": ["moleculekit/fileformats/xtc/include", "moleculekit/fileformats/xtc"],
}


REFERENCE = os.environ.get("MKB_REFERENCE_SRC", "")


def ref_available(reference: str = REFERENCE) -> bool:
    return bool(reference) and all(os.path.isfile(os.path.join(reference, p)) for p in MODULES.values())


def built() -> bool:
    return all(os.path.isfile(os.path.join(OUT, f"{m}.so")) for m in MODULES)


def build(reference: str = REFERENCE, force: bool = False, verbose: bool = True) -> bool:
    """Returns True if oracle/_ref holds both modules after the call."""
    if built() and not force:
        return True
    if not ref_available(reference):
        return False
    import numpy

    os.makedirs(OUT, exist_ok=True)
    pyinc = sysconfig.get_paths()["include"]
    npinc = numpy.get_include()
    tmp = tempfile.mkdtemp(prefix="mkb_ref_")
    try:
        for mod, rel in MODULES.items():
            src = os.path.join(reference, rel)
            cpp = os.path.join(tmp, f"{mod}.cpp")
            so = os.path.join(OUT, f"{mod}.so")
            incs = [os.path.join(reference, d) for d in EXTRA_INCLUDES.get(mod, [])]
            extra = [os.path.join(reference, f) for f in EXTRA_SOURCES.get(mod, [])]
            cmd1 = [sys.executable, "-m", "cython", "--cplus"] + [f"-I{d}" for d in incs] + [src, "-o", cpp]
            cmd2 = [
                "g++", "-O3", "-shared", "-fPIC", "-w",
                "-DPy_LIMITED_API=0x030B0000",
                "-DNPY_NO_DEPRECATED_API=NPY_1_7_API_VERSION",
                f"-I{pyinc}", f"-I{npinc}"] + [f"-I{d}" for d in incs] + [cpp] + extra + ["-o", so]
            for cmd in (cmd1, cmd2):
                if verbose:
                    print("[oracle/_ref]", " ".join(cmd), flush=True)
                subprocess.run(cmd, check=True, stdout=subprocess.DEVNULL if not verbose else None)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return built()


def load():
    """Import the reference extension modules from oracle/_ref.  Returns (occupancy_utils, distance_utils,
    bondguesser_utils) or None."""
    if not built():
        return None
    import importlib.util

    mods = []
    for mod in MODULES:
        path = os.path.join(OUT, f"{mod}.so")
        spec = importlib.util.spec_from_file_location(mod, path)
        m = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(m)
        mods.append(m)
    return tuple(mods)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=REFERENCE)
    ap.add_argument("--force", action="store_true")
    a = ap.parse_args()
    ok = build(a.reference, a.force)
    print("oracle/_ref built:", ok)
    sys.exit(0 if ok else 1)
