"""XTC writer and integer reader in plain Python -- TEST INFRASTRUCTURE ONLY (the package never imports it).

  moleculekit/fileformats/xtc/src/xdrfile.cpp       xdrfile_compress_coord_float (encoder), encodebits / encodeints,
                                                    sizeofint / sizeofints, the magicints table
  moleculekit/fileformats/xtc/src/xdrfile_xtc.cpp   the frame header (magic, natoms, step, time, box)

The product only decodes XTC (K11); nothing in it can write a stream.  This module writes one, so the decoder can be
tested on streams nobody committed: :func:`compress_frame` restates the reference writer's choices from the integer
lattice coordinates (it reproduces the committed files in tests/golden/xtc/ byte for byte), and :class:`Block` writes a
coordinate block through the same primitives with the choices left to the caller, for streams the reference's heuristic
never produces (9- and 10-atom runs, runs at small-range indices above 64, ranges of 2^31 or more).  :func:`read_ints`
is a third reading of the format, beside ``oracle_xtc_decode_block`` and the kernel: Python integers make the
mixed-radix arithmetic exact by construction.

A decoded coordinate is ``(float)int * (float)(1.0 / (double)precision)``: :func:`coords` computes it from integers.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

MAGIC = 1995
MAGICINTS = (0, 0, 0, 0, 0, 0, 0, 0, 0, 8, 10, 12, 16, 20, 25, 32, 40, 50, 64, 80, 101, 128, 161, 203, 256, 322, 406, 512, 645,
             812, 1024, 1290, 1625, 2048, 2580, 3250, 4096, 5060, 6501, 8192, 10321, 13003, 16384, 20642, 26007, 32768, 41285,
             52015, 65536, 82570, 104031, 131072, 165140, 208063, 262144, 330280, 416127, 524287, 660561, 832255, 1048576,
             1321122, 1664510, 2097152, 2642245, 3329021, 4194304, 5284491, 6658042, 8388607, 10568983, 13316085, 16777216)
FIRSTIDX, LASTIDX = 9, len(MAGICINTS)
MAXABS = 2**31 - 1 - 2  # INT_MAX - 2
INT_MAX = 2**31 - 1


def _i32(v: int) -> int:
    """v wrapped to a C int (two's complement), as the reference's int arithmetic leaves it"""
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v & 0x80000000 else v


def _iabs(v: int) -> int:
    """C abs() of an int result: abs(INT_MIN) stays INT_MIN"""
    v = _i32(v)
    return v if v == -(1 << 31) else abs(v)


def sizeofint(size: int) -> int:
    """bits of one size, at most 32 (xdrfile.cpp sizeofint)"""
    return min(int(size).bit_length(), 32)


def sizeofints(sizes) -> int:
    """bits of the product of the sizes (xdrfile.cpp sizeofints: whole low bytes plus the bits of the top byte)"""
    p = 1
    for s in sizes:
        p *= int(s)
    return p.bit_length()


# ------------------------------------------------------------------------------------------------ bit primitives
class BitWriter:
    """A bit stream, most significant bit first, as encodebits writes it into xdrfile's buffer."""

    def __init__(self):
        self._out = bytearray()
        self._acc = 0   # bits not yet moved to _out
        self._n = 0     # number of them
        self.nbits = 0  # bits written in all

    def send_bits(self, n: int, value: int) -> None:
        """the n low bits of value, most significant first"""
        value = int(value)
        if n < 0 or not 0 <= value < (1 << n):
            raise ValueError(f"{value} does not fit in {n} bits")
        self._acc = (self._acc << n) | value
        self._n += n
        self.nbits += n
        if self._n >= 256:
            r = self._n & 7
            self._out += (self._acc >> r).to_bytes((self._n - r) >> 3, "big")
            self._acc &= (1 << r) - 1
            self._n = r

    def send_ints(self, nbits: int, sizes, nums) -> None:
        """Three integers as one mixed-radix number ((nums[0]·sizes[1] + nums[1])·sizes[2] + nums[2]) in nbits bits:
        8-bit chunks, least significant first, then the remaining high bits (encodeints; the inverse of the decoder's
        receiveints / ``XtcBits::take3``)."""
        nums = [int(v) for v in nums]
        sizes = [int(v) for v in sizes]
        if not all(0 <= v < s for v, s in zip(nums, sizes)):
            raise ValueError(f"{nums} outside sizes {sizes}")
        value = (nums[0] * sizes[1] + nums[1]) * sizes[2] + nums[2]
        if value >> nbits:
            raise ValueError(f"mixed-radix value {value} does not fit in {nbits} bits")
        while nbits > 8:
            self.send_bits(8, value & 0xFF)
            value >>= 8
            nbits -= 8
        self.send_bits(nbits, value)

    def tobytes(self) -> bytes:
        """the stream, its last byte padded with zero bits"""
        r = (-self._n) & 7
        return bytes(self._out) + (self._acc << r).to_bytes((self._n + r) >> 3, "big")


class BitReader:
    """MSB-first reader over one coordinate block; reading past its end is an error."""

    def __init__(self, data: bytes):
        self.data = bytes(data)
        self.pos = 0

    def take(self, n: int) -> int:
        if n == 0:
            return 0
        end = self.pos + n
        if end > 8 * len(self.data):
            raise ValueError("coordinate block ends inside a field")
        a, b = self.pos >> 3, (end + 7) >> 3
        v = int.from_bytes(self.data[a:b], "big") >> (8 * b - end)
        self.pos = end
        return v & ((1 << n) - 1)

    def take_ints(self, nbits: int, sizes) -> list:
        value, shift = 0, 0
        while nbits > 8:
            value |= self.take(8) << shift
            shift += 8
            nbits -= 8
        value |= self.take(nbits) << shift
        n2 = value % sizes[2]
        value //= sizes[2]
        return [value // sizes[1], value % sizes[1], n2]


def xdr_int(*v) -> bytes:
    return b"".join(struct.pack(">i", _i32(int(x))) for x in v)


def xdr_float(*v) -> bytes:
    return np.asarray(v, dtype=np.float32).astype(">f4").tobytes()


def xdr_opaque(data: bytes) -> bytes:
    """opaque bytes padded with zeros to a multiple of 4 (xdr_opaque)"""
    return bytes(data) + bytes((-len(data)) & 3)


# ------------------------------------------------------------------------------------------------ one coordinate block
class Block:
    """One frame's compressed coordinate block, written the way ``xdrfile_decompress_coord_float`` reads it.

    The block keeps the decoder's state -- the small-range index and the current run length -- so every call is checked
    against what a decoder will read, and it records in ``cover`` (a set) which decoder branches the block drives."""

    def __init__(self, minint, maxint, smallidx: int, cover: set | None = None):
        self.minint = [int(v) for v in minint]
        self.maxint = [int(v) for v in maxint]
        self.sizeint = [(b - a + 1) & 0xFFFFFFFF for a, b in zip(self.minint, self.maxint)]
        if not all(self.sizeint):
            raise ValueError("a range of 2^32 values has no size")
        if not FIRSTIDX <= smallidx < LASTIDX:
            raise ValueError(f"smallidx {smallidx} outside the table")
        self.cover = set() if cover is None else cover
        if max(self.sizeint) > 0xFFFFFF:
            self.bitsizeint = [sizeofint(s) for s in self.sizeint]
            self.bitsize = 0
            self.cover.add(("wide_axes", sum(s > 0xFFFFFF for s in self.sizeint)))
        else:
            self.bitsize = sizeofints(self.sizeint)
        if any(b - a + 1 > INT_MAX for a, b in zip(self.minint, self.maxint)):
            self.cover.add(("range_overflows_int",))
        if min(self.minint) < 0:
            self.cover.add(("negative_minint",))
        self.smallidx0 = self.smallidx = int(smallidx)
        self.run = 0      # the decoder's run length (3 x atoms); a flag-less atom repeats it
        self.atoms = []   # lattice coordinates in the order the decoder emits them
        self.bits = BitWriter()

    @property
    def smallnum(self) -> int:
        return MAGICINTS[self.smallidx] // 2

    def group(self, full, run=(), is_smaller: int = 0, flag: bool | None = None) -> None:
        """One pass of the decoder's loop: the full-range triple ``full``, the flag bit (with the 5-bit code
        ``3·len(run) + is_smaller + 1`` when set), one small triple per atom of ``run`` at the current small range, then
        the small-range step ``is_smaller``.  ``run`` holds lattice coordinates: the first is coded against ``full`` and
        emitted before it, every later one against its predecessor.  ``flag=None`` sends the flag only when the decoder
        needs it (a new run length or a step)."""
        full = [int(v) for v in full]
        run = [[int(v) for v in a] for a in run]
        n3 = 3 * len(run)
        if flag is None:
            flag = n3 != self.run or is_smaller != 0
        if not flag and (n3 != self.run or is_smaller != 0):
            raise ValueError("without a flag the decoder repeats the last run and keeps its small range")
        if not -1 <= is_smaller <= 1 or n3 + is_smaller + 1 > 31 or n3 + is_smaller + 1 < 0:
            raise ValueError(f"no 5-bit code for a run of {len(run)} atoms and step {is_smaller}")
        if not FIRSTIDX <= self.smallidx + is_smaller < LASTIDX:
            raise ValueError("the step leaves the small-range table")
        rel = [(v - a) & 0xFFFFFFFF for v, a in zip(full, self.minint)]
        if not all(r < s for r, s in zip(rel, self.sizeint)):
            raise ValueError(f"{full} outside [minint, maxint]")
        if self.bitsize == 0:
            for d in range(3):
                self.bits.send_bits(self.bitsizeint[d], rel[d])
        else:
            self.bits.send_ints(self.bitsize, self.sizeint, rel)
            self.cover.add(("full_bits", "<=32" if self.bitsize <= 32 else "33-64" if self.bitsize <= 64 else ">64"))
            value = (rel[0] * self.sizeint[1] + rel[1]) * self.sizeint[2] + rel[2]
            if value in (2**32 - 1, 2**32, 2**64 - 1, 2**64):  # where a decoder's 32- / 64-bit arithmetic ends
                self.cover.add(("full_value", value))
        if flag:
            code = n3 + is_smaller + 1
            self.bits.send_bits(1, 1)
            self.bits.send_bits(5, code)
            self.run = n3
            if n3:
                self.cover.add(("run_code", code))
        else:
            self.bits.send_bits(1, 0)
            if n3:
                self.cover.add(("flagless_run",))
        size = MAGICINTS[self.smallidx]
        prev = full
        for a in run:
            self.bits.send_ints(self.smallidx, (size, size, size), [_i32(a[d] - prev[d] + self.smallnum) for d in range(3)])
            self.cover.add(("run_smallidx", self.smallidx))
            prev = a
        self.atoms += ([run[0], full] + run[1:]) if run else [full]
        if is_smaller:
            self.smallidx += is_smaller
            self.cover.add(("adapted_to", self.smallidx))

    def tobytes(self, precision) -> bytes:
        """precision, minint, maxint, smallidx, the byte count and the padded stream (xdrfile.cpp block layout)"""
        data = self.bits.tobytes()
        self.cover.add(("block_header", float(np.float32(precision)), tuple(self.minint), tuple(self.maxint),
                        self.smallidx0))
        return (xdr_float(precision) + xdr_int(*self.minint) + xdr_int(*self.maxint) + xdr_int(self.smallidx0) +
                xdr_int(len(data)) + xdr_opaque(data))


def to_lattice(xyz, precision) -> np.ndarray:
    """The reference writer's float -> int step: lf = x·precision in float32, ± 0.5 in float32, truncated."""
    x = np.asarray(xyz, dtype=np.float32)
    lf = x * np.float32(precision)
    lf = np.where(x >= 0, lf + np.float32(0.5), lf - np.float32(0.5)).astype(np.float32)
    if np.any(np.abs(lf.astype(np.float64)) > MAXABS):
        raise ValueError("Internal overflow compressing coordinates")
    return lf.astype(np.int64)


def compress_frame(ints, precision, cover: set | None = None) -> bytes:
    """``xdrfile_compress_coord_float`` from the lattice coordinates ``ints`` (natoms > 9, 3): the coordinate block after
    the atom count.  Every choice is the reference writer's, including its C int arithmetic (the overflow of the squared
    run distance at large small ranges).  Where the reference would print "Internal overflow" or read past its table,
    this raises."""
    c = [[int(v) for v in a] for a in np.asarray(ints).reshape(-1, 3)]
    n = len(c)
    if n <= 9:
        raise ValueError("nine atoms or fewer are written as plain floats")
    minint = [min(a[d] for a in c) for d in range(3)]
    maxint = [max(a[d] for a in c) for d in range(3)]
    if any(np.float32(b) - np.float32(a) >= np.float32(MAXABS) for a, b in zip(minint, maxint)):
        raise ValueError("Internal overflow compressing coordinates")
    mindiff = INT_MAX
    for a, b in zip(c, c[1:]):
        diff = _i32(_iabs(a[0] - b[0]) + _iabs(a[1] - b[1]) + _iabs(a[2] - b[2]))
        mindiff = min(mindiff, diff)
    smallidx = FIRSTIDX
    while smallidx < LASTIDX and MAGICINTS[smallidx] < mindiff:
        smallidx += 1
    maxidx = min(LASTIDX, smallidx + 8)
    if maxidx >= LASTIDX:
        raise ValueError(f"initial smallidx {smallidx}: the reference reads magicints[{maxidx}], past its table")
    minidx = maxidx - 8
    larger = MAGICINTS[maxidx] // 2
    blk = Block(minint, maxint, smallidx, cover)
    smaller = MAGICINTS[max(FIRSTIDX, smallidx - 1)] // 2
    prevrun, prev, i = -1, None, 0
    while i < n:
        this = c[i]
        if blk.smallidx < maxidx and i >= 1 and all(_iabs(this[d] - prev[d]) < larger for d in range(3)):
            is_smaller = 1
        elif blk.smallidx > minidx:
            is_smaller = -1
        else:
            is_smaller = 0
        smallnum = blk.smallnum
        is_small = i + 1 < n and all(_iabs(this[d] - c[i + 1][d]) < smallnum for d in range(3))
        if is_small:  # the first two atoms trade places: water O then H compresses better
            c[i], c[i + 1] = c[i + 1], c[i]
        full = prev = c[i]
        i += 1
        run = []
        if not is_small and is_smaller == -1:
            is_smaller = 0
        while is_small and len(run) < 8:
            this = c[i]
            tmpsum = 0
            for d in range(3):
                tmpsum = _i32(tmpsum + _i32((this[d] - prev[d]) * (this[d] - prev[d])))
            if is_smaller == -1 and tmpsum >= _i32(smaller * smaller):
                is_smaller = 0
            run.append(this)
            prev = this
            i += 1
            is_small = i < n and all(_iabs(c[i][d] - prev[d]) < smallnum for d in range(3))
        flag = 3 * len(run) != prevrun or is_smaller != 0
        if flag:
            prevrun = 3 * len(run)
        blk.group(full, run, is_smaller, flag)
        if is_smaller < 0:
            smaller = MAGICINTS[blk.smallidx - 1] // 2
        elif is_smaller > 0:
            smaller = smallnum
    return blk.tobytes(precision)


# ------------------------------------------------------------------------------------------------ frames and files
@dataclass
class Frame:
    """One XTC frame.  ``xyz`` (natoms, 3) float32 for the plain branch (natoms <= 9), else the lattice coordinates
    ``ints`` (natoms, 3) at ``precision``; :func:`read_ints` also fills the block header it read."""
    step: int = 0
    time: float = 0.0
    box: np.ndarray = field(default_factory=lambda: np.zeros((3, 3), np.float32))
    precision: float | None = None
    ints: np.ndarray | None = None
    xyz: np.ndarray | None = None
    minint: tuple | None = None
    maxint: tuple | None = None
    smallidx: int | None = None
    block: bytes | None = None  # a ready-made coordinate block (from :class:`Block`) instead of compress_frame's

    @property
    def natoms(self) -> int:
        return len(self.xyz if self.xyz is not None else self.ints)


def frame_bytes(fr: Frame, cover: set | None = None) -> bytes:
    """magic, natoms, step, time, the 9 box floats, natoms again, then the coordinates (xdrfile_xtc.cpp write_xtc)"""
    n = fr.natoms
    head = xdr_int(MAGIC, n, fr.step) + xdr_float(fr.time) + xdr_float(*np.asarray(fr.box, np.float32).ravel()) + xdr_int(n)
    if n <= 9:
        if fr.xyz is None:
            raise ValueError("nine atoms or fewer are written as plain floats: give xyz")
        if cover is not None:
            cover.add(("plain",))
        return head + np.asarray(fr.xyz, np.float32).astype(">f4").tobytes()
    precision = np.float32(fr.precision)
    if cover is not None:
        cover.add(("precision", float(precision)))
        cover.add(("natoms", n))
    if fr.block is not None:
        return head + fr.block
    return head + compress_frame(fr.ints, precision, cover)


def write_frames(frames, cover: set | None = None) -> bytes:
    return b"".join(frame_bytes(fr, cover) for fr in frames)


def write_xtc(coords, box, time, step, precision=1000.0) -> bytes:
    """The bytes of the reference's ``write_xtc(filename, coords, box, time, step)`` (xtc.pyx): coords (natoms, 3, F)
    float32 in nm, box (3, 3, F), time (F,), step (F,), every frame at ``precision``."""
    coords = np.asarray(coords, np.float32)
    precision = precision if precision > 0 else 1000.0  # the reference's rule, applied before the float -> int step
    frames = []
    for f in range(coords.shape[2]):
        xyz = coords[:, :, f]
        fr = Frame(step=int(step[f]), time=np.float32(time[f]), box=np.asarray(box, np.float32)[:, :, f])
        if len(xyz) <= 9:
            fr.xyz = xyz
        else:
            fr.precision, fr.ints = precision, to_lattice(xyz, precision)
        frames.append(fr)
    return write_frames(frames)


# ------------------------------------------------------------------------------------------------ reading
def _decode_block(data: bytes, natoms: int, minint, maxint, smallidx: int) -> np.ndarray:
    sizeint = [(b - a + 1) & 0xFFFFFFFF for a, b in zip(minint, maxint)]
    if not all(sizeint):
        raise ValueError("zero size")
    wide = max(sizeint) > 0xFFFFFF
    bitsizeint = [sizeofint(s) for s in sizeint]
    bitsize = sizeofints(sizeint)
    if not FIRSTIDX <= smallidx < LASTIDX:
        raise ValueError(f"smallidx {smallidx} outside the table")
    r = BitReader(data)
    out, run = [], 0
    while len(out) < natoms:
        rel = [r.take(b) for b in bitsizeint] if wide else r.take_ints(bitsize, sizeint)
        cur = [_i32(v + a) for v, a in zip(rel, minint)]
        is_smaller = 0
        if r.take(1):
            code = r.take(5)
            run, is_smaller = code - code % 3, code % 3 - 1
        prev = cur
        size = MAGICINTS[smallidx]
        for k in range(run // 3):
            s = r.take_ints(smallidx, (size, size, size))
            s = [_i32(v + p - size // 2) for v, p in zip(s, prev)]
            out += [s, cur] if k == 0 else [s]
            prev = s
        if not run:
            out.append(cur)
        smallidx += is_smaller
        if not FIRSTIDX <= smallidx < LASTIDX:
            raise ValueError("the small range left the table")
    if len(out) != natoms:
        raise ValueError("a run crosses the end of the frame")
    return np.array(out, dtype=np.int64).reshape(natoms, 3)


def read_ints(raw: bytes) -> list:
    """Every frame of an XTC byte string as a :class:`Frame`: its header and the integer lattice coordinates (or the
    plain floats of a frame of nine atoms or fewer)."""
    raw = bytes(raw)
    pos, frames = 0, []
    while pos < len(raw):
        magic, natoms, step = struct.unpack_from(">iii", raw, pos)
        if magic != MAGIC:
            raise ValueError(f"bad magic {magic} at byte {pos}")
        time = np.frombuffer(raw, ">f4", 1, pos + 12).astype(np.float32)[0]
        box = np.frombuffer(raw, ">f4", 9, pos + 16).astype(np.float32).reshape(3, 3)
        (n2,) = struct.unpack_from(">i", raw, pos + 52)
        if n2 != natoms:
            raise ValueError("the two atom counts of a frame differ")
        pos += 56
        fr = Frame(step=step, time=time, box=box)
        if natoms <= 9:
            fr.xyz = np.frombuffer(raw, ">f4", 3 * natoms, pos).astype(np.float32).reshape(natoms, 3)
            pos += 12 * natoms
        else:
            fr.precision = np.frombuffer(raw, ">f4", 1, pos).astype(np.float32)[0]
            h = struct.unpack_from(">8i", raw, pos + 4)
            fr.minint, fr.maxint, fr.smallidx, nbytes = h[0:3], h[3:6], h[6], h[7]
            if nbytes < 0 or pos + 36 + nbytes > len(raw):
                raise ValueError("truncated coordinate block")
            fr.ints = _decode_block(raw[pos + 36:pos + 36 + nbytes], natoms, fr.minint, fr.maxint, fr.smallidx)
            pos += 36 + nbytes + ((-nbytes) & 3)
        frames.append(fr)
    return frames


def coords(frames) -> np.ndarray:
    """(natoms, 3, F) float32 as a decoder returns them: (float)int · (float)(1.0 / (double)precision), one float32
    rounding per step, or the plain floats"""
    out = []
    for fr in frames:
        if fr.xyz is not None:
            out.append(np.asarray(fr.xyz, np.float32))
        else:
            inv = np.float32(1.0 / np.float64(np.float32(fr.precision)))
            out.append(np.asarray(fr.ints).astype(np.float32) * inv)
    return np.ascontiguousarray(np.stack(out, axis=2)) if out else np.zeros((0, 3, 0), np.float32)
