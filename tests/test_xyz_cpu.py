"""The host side of XYZ trajectory reading and writing (moleculekit_b200/xyz.py; K26 indexes, parses and formats on the
device): the independent oracle's round trip and a small file byte by byte, the writer's argument and range checks that
run before the file is opened, the C-ABI symbols, and K26's decimal conversion (csrc/xyz_number.cuh) built with the
host compiler and held to float() token by token."""
import os
import random
import shutil
import subprocess

import numpy as np
import pytest

from oracle import xyz_format as of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(N, F, seed, scale=30.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def test_oracle_round_trip():
    for N in (1, 2, 5):
        el = ["C", "Hx", "O"] * 2
        el = el[:N]
        xs = frames(N, 4, N)
        raw = of.write(xs, el, comment="round trip")
        got = of.read(raw)
        assert got["natoms"] == N and got["element"] == el and got["comment"] == "round trip"
        want = np.float32([[[float("%15.8f" % v) for v in row] for row in x] for x in xs])
        assert np.array_equal(got["coords"], want)
        # the file's own values come back unchanged
        assert of.write(list(got["coords"]), el, "round trip") == raw


def test_two_atoms_byte_by_byte():
    xs = [np.float32([[1.0, -2.5, 0.0625], [123456.125, -0.0, 99999.5]])]
    want = (b"2\nt\n"
            b"C       1.00000000     -2.50000000      0.06250000\n"
            b"Na 123456.12500000     -0.00000000  99999.50000000\n")
    assert of.write(xs, ["C", "Na"], comment="t") == want
    from moleculekit_b200 import xyz as px

    assert px.frame_bytes(2, b"2\nt\n", 2) == len(want)


def test_writer_argument_checks(tmp_path):
    import torch
    from moleculekit_b200 import _lib
    from moleculekit_b200 import xyz as px

    c = np.zeros((6, 3, 4), np.float32)
    el = ["C"] * 6

    def huge(v, at=(5, 1, 2)):
        x = c.copy()
        x[at] = v
        return x

    cases = [((c[:, :2], el), {}), ((c[0], el), {}), ((np.zeros((0, 3, 4), np.float32), []), {}),
             ((c, el[:5]), {}), ((c, "CCCCCC"), {}), ((c, el[:5] + [""]), dict(match="atom 5")),
             ((c, el[:5] + ["C a"]), dict(match="atom 5")), ((c, el[:5] + ["é"]), dict(match="atom 5")),
             ((c, el[:5] + ["C\x1c"]), dict(match="atom 5")), ((c, el[:5] + [7]), dict(match="atom 5")),
             ((c, el[:5] + ["X" * 257]), dict(match="atom 5")),
             ((c, el), dict(comment="a\nb")), ((c, el), dict(comment="a\rb")), ((c, el), dict(comment="café")),
             ((c, el), dict(comment=b"bytes")), ((c, el), dict(chunk_bytes=0))]
    for v in (np.nan, np.inf, -np.inf, 1e6, np.float32(-100000.0), np.nextafter(np.float32(1e6), np.float32(0)) * 2):
        cases.append(((huge(v), el), dict(match="frame 2, atom 5, axis y")))
    x = huge(1e7, (4, 0, 1))
    x[3, 2, 1] = np.nan
    x[0, 0, 3] = -5e5
    cases.append(((x, el), dict(match="frame 1, atom 3, axis z")))
    for args, kw in cases:
        match = kw.pop("match", None)
        with pytest.raises(ValueError, match=match):
            px.xyz_bytes(*args, **kw)
        fn = tmp_path / "untouched.xyz"
        with pytest.raises(ValueError, match=match):
            px.write_xyz(str(fn), *args, **kw)
        assert not fn.exists()
    # the range rule's edges pass the checks: only the missing device stops the call
    edge = huge(np.float32(999999.9375), (0, 0, 0))
    edge[1, 1, 1] = np.float32(-99999.9921875)
    edge[2, 2, 2] = np.float32(-0.0)
    if not torch.cuda.is_available():
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            px.xyz_bytes(edge, el)
        fn = tmp_path / "t.xyz"
        fn.write_bytes(of.write(frames(3, 2, 0), ["H"] * 3))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            px.read_xyz_device(str(fn))
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            px.decode_xyz_device(torch.zeros(16, dtype=torch.uint8), 1, np.zeros(0), 3)
    with pytest.raises(_lib.MkbError, match="no CPU fallback"):
        px.encode_xyz_device(torch.zeros((6, 3, 4)), el)
    # no frames: an empty file, no device needed
    assert px.xyz_bytes(np.zeros((5, 3, 0), np.float32), ["H"] * 5, comment="empty") == b""


def test_reader_rejects_before_the_device(tmp_path):
    from moleculekit_b200 import xyz as px

    for raw, match in ((b"", "no frames"), (b"  \n\t\n", "no frames"), (b"x\ncomment\n", "line 1, column 1: the atom "
                       "count line 'x' does not start with an integer"), (b"0\n\n", "atom count must be 1"),
                       (b"\xff\n", "line 1, column 1: the line is not UTF-8")):
        fn = tmp_path / "r.xyz"
        fn.write_bytes(raw)
        with pytest.raises(ValueError, match=match):
            px.index_xyz(str(fn))
    with pytest.raises(ValueError, match="chunk_bytes"):
        px.index_xyz(str(fn), chunk_bytes=0)


def test_abi_symbols():
    from moleculekit_b200 import _lib, build

    build.build(verbose=False)
    lib = _lib.load()
    hdr = open(os.path.join(ROOT, "include", "mkb200.h")).read()
    for name, nargs in (("mkb_xyz_index", 11), ("mkb_xyz_decode", 13), ("mkb_xyz_encode", 12)):
        assert name in _lib.EXPORTS and hasattr(lib, name)
        assert len(getattr(lib, name).argtypes) == nargs
        decl = hdr[hdr.index(f"int {name}("):]
        assert decl[:decl.index(");")].count(",") + 1 == nargs


HARNESS = r"""
#include <cstdio>
#include <iostream>
#include <string>
#include "xyz_number.cuh"
struct Rd { const unsigned char *b; long long end; unsigned at(long long p) const { return p < end ? b[p] : '\n'; } };
int main() {
    std::string s;
    while (std::getline(std::cin, s)) {
        Rd r{(const unsigned char *)s.data(), (long long)s.size()};
        long long p = 0;
        unsigned bits = 0;
        if (mkb::xyz_number(r, p, bits) && p == (long long)s.size()) printf("%08x\n", bits);
        else printf("host\n");
    }
}
"""


def random_tokens(n, seed):
    """decimal tokens of 1-25 digits, exponents -330 ... 310, signs, points anywhere"""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        d = "".join(rng.choice("0123456789") for _ in range(rng.randint(1, 25)))
        if rng.random() < 0.4:
            k = rng.randint(0, len(d))
            d = d[:k] + "." + d[k:]
        sign = rng.choice(["", "", "-", "+"])
        exp = rng.choice("eE") + str(rng.randint(-330, 310)) if rng.random() < 0.6 else ""
        out.append(sign + d + exp)
    return out


def test_conversion_host_build_matches_float(tmp_path):
    """xyz_number.cuh built by the host compiler: every token it decides is np.float32(float(token)) bit for bit, and
    it leaves to the host exactly the undecided and out-of-grammar tokens"""
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no host C++ compiler")
    exe = tmp_path / "conv"
    src = tmp_path / "conv.cpp"
    src.write_text(HARNESS)
    subprocess.run([cxx, "-O2", "-std=c++17", f"-I{os.path.join(ROOT, 'moleculekit_b200', 'csrc')}", str(src), "-o",
                    str(exe)], check=True)
    special = ["1.00000005960464477539062500001", "nan", "-nan", "NaN", "+inf", "-Infinity", "iNfInItY", "1e39",
               "-1e39", "1e-46", "1.4e-45", "-0.0", "+0.0", ".5", "5.", "+.5e+1", "1E+02", "4.9406564584124654e-324",
               "2.4703282292062328e-324", "1.7976931348623157e308", "1.7976931348623159e308", "0." + "0" * 400 + "1e400",
               "1" + "0" * 400 + "e-400", "3.4028235677973366e38", "00012.5000", "1e-99999999999", "0e999999999"]
    host_only = ["9007199254740993.00000000001", "1_0", "1e", ".", "e5", "1.2.3", "0x10", "nana", "infinit", "1e+",
                 "--1", "1,5", "١"]
    toks = special + host_only + random_tokens(100000, 26)
    out = subprocess.run([str(exe)], input="\n".join(toks) + "\n", capture_output=True, text=True,
                         check=True).stdout.split()
    assert len(out) == len(toks)
    for t, o in zip(toks, out):
        if t in host_only:
            assert o == "host", t
        elif o != "host":
            with np.errstate(over="ignore"):
                want = np.array([float(t)]).astype(np.float32).view(np.uint32)[0]
            assert int(o, 16) == int(want), (t, o, hex(want))
    assert out[0] == "3f800000"  # rounded twice: to the double 1 + 2^-24, then to even
    assert out[2] == "ffc00000"
    assert sum(o == "host" for o in out[len(special) + len(host_only):]) < 100
