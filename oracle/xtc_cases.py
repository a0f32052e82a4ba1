"""Seeded XTC streams for the decoder tests -- TEST INFRASTRUCTURE ONLY.

Every case is a list of :class:`oracle.xtc_writer.Frame` (integer lattice coordinates, or plain floats for nine atoms or
fewer), the file written from them and the set of decoder branches the writer drove (``cover``).  The expected decoded
coordinates follow from the integers alone (:func:`oracle.xtc_writer.coords`), so a decoder is compared bit for bit.

Most cases go through the reference writer's own heuristic (:func:`oracle.xtc_writer.compress_frame`); the ones named in
``PRIMITIVE`` are built group by group with :class:`oracle.xtc_writer.Block`, for what that heuristic never writes: runs
of 9 and 10 atoms (codes 27-31), runs at small-range indices 65-72, the small range walked down to 9 and up to 72, and
ranges of 2^31 lattice steps or more.  The whole set is about 4·10^5 atom-frames and takes seconds to write.
"""
from __future__ import annotations

import zlib
from dataclasses import dataclass

import numpy as np

from oracle import xtc_writer as xw

INT_MIN, INT_MAX = -(2**31), 2**31 - 1


@dataclass
class Case:
    name: str
    frames: list
    raw: bytes
    cover: set

    def expected(self) -> np.ndarray:
        return xw.coords(self.frames)


def _rng(name: str):
    return np.random.default_rng(zlib.crc32(name.encode()))


def _headers(frames):
    """distinct step / time / box per frame, so a decoder that mixes frames up shows it"""
    for f, fr in enumerate(frames):
        fr.step, fr.time = 10 * f + 5, np.float32(0.5 * f + 1)
        fr.box = (np.diag([3.1, 3.2, 3.3]) + 0.01 * f).astype(np.float32)
    return frames


def _water(rng, nw, L):
    """(3·nw, 3) float nm: O at random in a box of side L, two H within ~0.1 nm"""
    o = rng.uniform(0, L, size=(nw, 1, 3))
    return np.concatenate([o, o + rng.normal(0, 0.06, size=(nw, 2, 3))], axis=1).reshape(-1, 3)


def _float_frames(xyz_frames, precision):
    """frames from float32 coordinates through the reference writer's float -> int step"""
    out = []
    for xyz in xyz_frames:
        xyz = np.asarray(xyz, np.float32)
        if len(xyz) <= 9:
            out.append(xw.Frame(xyz=xyz))
        else:
            out.append(xw.Frame(precision=precision, ints=xw.to_lattice(xyz, precision)))
    return out


def _paired(rng, lo, hi, n, near=3):
    """(n, 3) lattice points uniform in [lo, hi] per axis, every second one within `near` steps of its predecessor
    (keeps the writer's first small range low however wide the frame), with both corners present so the ranges are
    exactly [lo, hi]"""
    lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
    a = rng.integers(lo, hi + 1, size=(n, 3))
    a[1::2] = np.clip(a[0:-1:2] + rng.integers(-near, near + 1, size=a[1::2].shape), lo, hi)
    a[0], a[n // 2] = lo, hi
    return a


def _radix_atoms(rng, bits):
    """Lattice points whose full-range mixed-radix value sits at the edges a decoder splits on: 0, the largest value,
    and 2^32 - 1 / 2^32 / 2^63 / 2^64 - 1 / 2^64 where the product of the sizes allows them.  Sizes are chosen so the
    product has exactly `bits` bits."""
    s = min(int(round((2**bits - 1) ** (1 / 3))), 0xFFFFFF)
    while s * s * s > 2**bits - 1:
        s -= 1
    sizes = (s, s, min((2**bits - 1) // (s * s), 0xFFFFFF))
    prod = sizes[0] * sizes[1] * sizes[2]
    assert xw.sizeofints(sizes) == bits and max(sizes) <= 0xFFFFFF
    vals = [0, prod - 1] + [v for v in (2**32 - 1, 2**32, 2**63, 2**64 - 1, 2**64) if v < prod]
    lo = rng.integers(-(2**20), 2**20, size=3)
    pts = []
    for v in vals:
        n2 = v % sizes[2]
        t = v // sizes[2]
        pts.append(lo + np.array([t // sizes[1], t % sizes[1], n2]))
    # a far-apart filler after every edge point (neighbouring edge values are neighbouring lattice points, which the
    # writer would pair into a run), up to 20 atoms ending in a repeated atom so the first small range stays low
    fill = lo + rng.integers(0, np.array(sizes), size=(20 - len(pts), 3))
    fill[-1] = fill[-2]
    out = [a for p, q in zip(pts, fill) for a in (p, q)] + list(fill[len(pts):])
    return np.array(out, dtype=np.int64)


def _offset_walk(rng, prev, smallidx, lo, hi, extreme=0.25):
    """the next run atom after `prev` at small range `smallidx`, inside [lo, hi]; with probability `extreme` at the
    largest or smallest small offset on every axis (the largest mixed-radix value of that range)"""
    size = xw.MAGICINTS[smallidx]
    half = size // 2
    for _ in range(1000):
        if rng.random() < extreme:
            raw = np.full(3, size - 1 if rng.random() < 0.5 else 0)
        else:
            raw = rng.integers(0, size, size=3)
        a = prev + raw - half
        if np.all((a >= lo) & (a <= hi)):
            return a
    raise RuntimeError("no run atom fits")


def _plan_block(rng, smallidx, plan, lo, hi, precision, cover, fulls=None):
    """A coordinate block from a plan of groups (run atoms, small-range step, flag or None): full atoms uniform in
    [lo, hi] (or taken from `fulls`), run atoms a small-range step from their predecessor.  Returns the Frame."""
    lo, hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)
    groups, idx, k = [], smallidx, 0
    for nrun, step, flag in plan:
        full = fulls[k] if fulls is not None and k < len(fulls) else rng.integers(lo, hi + 1)
        k += 1
        run, prev = [], full
        for _ in range(nrun):
            prev = _offset_walk(rng, prev, idx, lo, hi)
            run.append(prev)
        groups.append((full, run, step, flag))
        idx += step
    atoms = np.array([a for g in groups for a in [g[0], *g[1]]])
    blk = xw.Block(atoms.min(0), atoms.max(0), smallidx, cover)
    for full, run, step, flag in groups:
        blk.group(full, run, step, flag)
    return xw.Frame(precision=precision, ints=np.array(blk.atoms, np.int64), block=blk.tobytes(precision))


# ------------------------------------------------------------------------------------------------ the cases
def _precision(p):
    def build(rng):
        xyz = [np.concatenate([_water(rng, 40, 4.0), rng.normal(0, 1.5, size=(80, 3))]) for _ in range(2)]
        return _float_frames(xyz, p)
    return build


def _natoms(n):
    def build(rng):
        return _float_frames([rng.normal(0, 1, size=(n, 3)) for _ in range(3)], 1000.0)
    return build


def _nframes(F):
    def build(rng):
        w = _water(rng, 8, 2.0)
        return _float_frames([w + rng.normal(0, 0.05, size=w.shape) * np.sqrt(f + 1) for f in range(F)], 1000.0)
    return build


def _wide(naxes):
    def build(rng):
        hi = np.array([2500, 1800, 3000]); hi[:naxes] = [21_000_000, 40_000_000, 17_000_000][:naxes]
        return [xw.Frame(precision=1000.0, ints=_paired(rng, -hi, hi, 80)) for _ in range(2)]
    return build


def _full_65_72(rng):
    """full-range triples of 65-72 bits: sizes about 2^22 .. 2^24 - 1 on all three axes, atoms close in pairs"""
    out = []
    for half in (2_700_000, 4_200_000, 8_388_607):
        lo = -half + rng.integers(-5, 5, size=3)
        out.append(xw.Frame(precision=1000.0, ints=_paired(rng, lo, lo + 2 * half, 120)))
    return out


def _radix_boundary(rng):
    return [xw.Frame(precision=1000.0, ints=_radix_atoms(rng, b)) for b in (32, 33, 64, 65, 72)]


def _water_runs(rng):
    w = _water(rng, 150, 3.0)
    return _float_frames([w + np.cumsum(rng.normal(0, 0.03, size=(4, *w.shape)), axis=0)[f] for f in range(4)], 1000.0)


def _chain(rng):
    """a smooth chain whose bond length swells and shrinks: long runs, the small range stepping up and down"""
    n = 2000
    scale = 0.004 * np.exp(2.5 * np.sin(np.linspace(0, 6 * np.pi, n)))[:, None]
    out = []
    for _ in range(3):
        out.append(np.cumsum(rng.normal(0, 1, size=(n, 3)) * scale, axis=0) - 1.0)
    return _float_frames(out, 1000.0)


def _mixed_headers(rng):
    """one file whose frames differ in precision, ranges and first small range"""
    frames = []
    for p, spread in ((1000.0, 1.5), (100.0, 40.0), (1e5, 0.3), (333.3, 6.0), (1000.0, 0.02)):
        xyz = np.concatenate([_water(rng, 20, spread), rng.normal(0, spread, size=(90, 3))])
        frames += _float_frames([xyz], p)
    return frames


def _large(rng):
    """50 000 atoms x 8 frames of water in a 8 nm box"""
    w = np.concatenate([_water(rng, 16_666, 8.0), rng.uniform(0, 8, size=(2, 3))])
    return _float_frames([w + rng.normal(0, 0.02 * (f + 1), size=w.shape) for f in range(8)], 1000.0)


def _runs_9_10(rng, cover):
    """runs of 9 and 10 atoms: codes 27, 28, 29, 30, 31, a flag-less repeated 10-atom run, then short runs"""
    plan = [(9, -1, None), (9, 0, True), (9, 1, None), (10, -1, None), (10, 0, True), (10, 0, False), (0, 0, None),
            (0, 0, False), (1, 1, None), (3, 0, None), (3, 0, False), (8, -1, None)]
    return [_plan_block(rng, 14, plan, [-5000] * 3, [5000] * 3, 1000.0, cover) for _ in range(2)]


def _high_smallidx(rng, cover):
    """runs at small-range indices 65..72 (mixed-radix run values of 65-72 bits), full triples of > 64 bits"""
    plan = [(2, 1, None)] * 7 + [(3, 0, None), (3, 0, False), (1, -1, None), (2, 1, None), (1, 0, None)]
    lo, hi = [-8_000_000] * 3, [8_000_000] * 3
    return [_plan_block(rng, 65, plan, lo, hi, 1000.0, cover) for _ in range(2)]


def _walk_9_72(rng, cover):
    """the small range walked from 40 down to 9, up to 72 and back to 60, one run atom per step"""
    plan = [(1, -1, None)] * 31 + [(1, 0, None)] + [(1, 1, None)] * 63 + [(2, 0, None), (2, 0, False)] + \
        [(1, -1, None)] * 12
    return [_plan_block(rng, 40, plan, [-30_000_000] * 3, [30_000_000] * 3, 1000.0, cover)]


def _range_2_31(rng, cover):
    """ranges of 2^31 lattice steps or more (32-bit fields with the top bit set), negative minint, and runs next to
    INT_MIN and INT_MAX where `prev - smallnum` and `value + minint` leave the int range before the result returns"""
    lo = np.array([INT_MIN + 2, -1_300_000_000, -70])
    hi = np.array([INT_MAX - 2, 1_100_000_000, 90])
    plan = [(1, 0, None), (0, 0, None), (2, 1, None), (0, 0, None), (1, 0, None), (1, 0, False)] + \
        [(0, 0, None), (1, -1, None)] * 3
    fulls = [lo, hi, lo + [1, 1, 1], hi - [1, 1, 1]]
    return [_plan_block(rng, 12, plan, lo, hi, p, cover, fulls) for p in (1000.0, 1e6)]


CASES = {f"precision_{p:g}": _precision(p) for p in (1, 10, 100, 1000, 1e4, 1e5, 1e6, 333.3)}
CASES.update({f"atoms_{n}": _natoms(n) for n in (9, 10, 11)})
CASES.update({f"frames_{F}": _nframes(F) for F in (1, 63, 64, 65, 300)})
CASES.update({f"wide_{k}axes": _wide(k) for k in (1, 2, 3)})
CASES.update(full_65_72=_full_65_72, radix_boundary=_radix_boundary, water=_water_runs, chain=_chain,
             mixed_headers=_mixed_headers, large=_large)
PRIMITIVE = dict(runs_9_10=_runs_9_10, high_smallidx=_high_smallidx, walk_9_72=_walk_9_72, range_2_31=_range_2_31)
NAMES = list(CASES) + list(PRIMITIVE)


def build(name: str) -> Case:
    rng, cover = _rng(name), set()
    frames = PRIMITIVE[name](rng, cover) if name in PRIMITIVE else CASES[name](rng)
    frames = _headers(frames)
    raw = xw.write_frames(frames, cover)
    cover.add(("frames", len(frames)))
    heads = [h for h in cover if h[0] == "block_header"]
    for what, key in (("precision", slice(1, 2)), ("ranges", slice(2, 4)), ("smallidx", slice(4, 5))):
        if len({h[key] for h in heads}) > 1:
            cover.add(("mixed", what))
    return Case(name, frames, raw, cover)
