"""The host side of multi-frame GRO reading and writing (moleculekit_b200/gro.py; K29 indexes, parses and formats on the
device): the independent oracle's round trip, the host prefix builder against the oracle writer's columns, the
writer's checks that run before the file is opened, and the reader's checks that run before the device."""
import numpy as np
import pytest

from oracle import gro_format as og


def frames(N, F, seed, scale=3.0):
    return [x for x in np.random.default_rng(seed).normal(0, scale, size=(F, N, 3)).astype(np.float32)]


def boxes(F, nine=False):
    out = []
    for f in range(F):
        b = np.diag(np.float32([5 + f, 6.5, 7.25]))
        if nine:
            b[1, 0], b[2, 0], b[2, 1] = 1.5, -0.25, 0.125 * f
        out.append(b)
    return out


def test_oracle_round_trip():
    for N, nine, vel in ((1, False, False), (3, True, True), (17, False, True)):
        top = og.random_topology(N, N)
        xs = frames(N, 4, N)
        vs = frames(N, 4, N + 1, 1.0) if vel else None
        raw = og.write(xs, top, boxes(4, nine), title="run", times=[0, 2.5, 5, 1000.25], steps=[0, 5, 10, 12345],
                       velocities=vs)
        got = og.read(raw)
        assert got["natoms"] == N and got["width"] == 8 and got["velocities"] == vel
        want = np.float32([[[float("%8.3f" % v) for v in row] for row in x] for x in xs])
        assert np.array_equal(got["coords"].view(np.uint32), want.view(np.uint32))
        if vel:
            wv = np.float32([[[float("%8.4f" % v) for v in row] for row in x] for x in vs])
            assert np.array_equal(got["vels"].view(np.uint32), wv.view(np.uint32))
        assert np.array_equal(got["box"], np.float32(boxes(4, nine)))
        assert got["time"].tolist() == [0, 2.5, 5, 1000.25] and got["step"].tolist() == [0, 5, 10, 12345]
        assert got["topology"]["resid"] == [r % 100000 for r in top["resid"]]
        assert got["topology"]["serial"] == [s % 100000 for s in top["serial"]]
        assert got["topology"]["resname"] == top["resname"] and got["topology"]["name"] == top["name"]
        # the file's own values come back unchanged
        again = og.write(list(got["coords"]), got["topology"], list(got["box"]), title="run",
                         times=got["time"], steps=got["step"], velocities=None if not vel else list(got["vels"]))
        assert again == raw
    # no time or step: NaN and -1
    got = og.read(og.write(frames(2, 2, 0), og.random_topology(2, 0), boxes(2), title="plain"))
    assert np.isnan(got["time"]).all() and (got["step"] == -1).all()


def test_prefix_matches_the_oracle_writer():
    from moleculekit_b200 import gro

    for N, seed in ((1, 0), (50, 1), (1000, 2)):
        top = og.random_topology(N, seed)
        raw = og.write(frames(N, 1, seed), top, boxes(1))
        lines = raw.split(b"\n")[2:2 + N]
        want = b"".join(ln[:20] for ln in lines)
        assert gro._prefix(gro._fields(top, N), N).tobytes() == want


def test_head_rows_match_the_oracle_writer():
    from moleculekit_b200 import gro

    N, F = 4, 5
    times, steps = [0.0, 1.5, -2.125, 10000.0, 3.0], [0, 7, 123456789, 2, 5]
    raw = og.write(frames(N, F, 3), og.random_topology(N, 3), boxes(F), title="Protein in water", times=times,
                   steps=steps)
    lines = raw.split(b"\n")
    rows = gro._head_rows("Protein in water", np.float64(times), np.int64(steps), N, F)
    for f in range(F):
        assert rows[f].tobytes() == lines[f * (N + 3)] + b"\n" + lines[f * (N + 3) + 1] + b"\n"


def _write_args(N=3, F=2):
    x = np.zeros((N, 3, F), np.float32)
    b = np.zeros((3, 3, F), np.float32)
    b[0, 0] = b[1, 1] = b[2, 2] = 3.0
    return x, b


@pytest.mark.parametrize("case, match", [
    ("nan", "coords at frame 1, atom 2, axis y is nan"),
    ("big", r"coords at frame 0, atom 1, axis z is 10000.0"),
    ("small", r"coords at frame 1, atom 0, axis x is -1000.0"),
    ("vel", r"velocities at frame 0, atom 0, axis x is 1000.0"),
    ("vinf", r"velocities at frame 1, atom 2, axis z is -inf"),
    ("box", r"box at frame 1, vector 1, axis x is 10000.0"),
    ("nobox", "box is required"),
    ("boxshape", r"box must be \(3, 3, F\)"),
    ("resname", "topology at atom 1, field resname is 'ABCDEF'"),
    ("name", "topology at atom 0, field name is 'C A'"),
    ("resid", "topology at atom 2, field resid is -1"),
    ("title", "title must be an ASCII str without a line break"),
    ("time", "time at frame 1 is not finite"),
    ("step", "step at frame 0 is not an integer"),
    ("chunk", "chunk_bytes must be positive"),
    ("shape", r"coords must be \(natoms, 3, F\)"),
])
def test_writer_checks_before_the_file_is_opened(tmp_path, case, match):
    from moleculekit_b200 import gro

    x, b = _write_args()
    kw = dict(topology={"resname": ["A", "B", "C"], "name": ["CA", "N", "O"], "resid": [1, 2, 3]}, box=b)
    if case == "nan":
        x[2, 1, 1] = np.nan
    elif case == "big":
        x[1, 2, 0] = 10000.0
    elif case == "small":
        x[0, 0, 1] = -1000.0
    elif case == "vel":
        v = np.zeros_like(x)
        v[0, 0, 0] = 1000.0
        kw["velocities"] = v
    elif case == "vinf":
        v = np.zeros_like(x)
        v[2, 2, 1] = -np.inf
        kw["velocities"] = v
    elif case == "box":
        b[1, 0, 1] = 10000.0
    elif case == "nobox":
        kw["box"] = None
    elif case == "boxshape":
        kw["box"] = np.zeros((3, 3))
    elif case == "resname":
        kw["topology"]["resname"][1] = "ABCDEF"
    elif case == "name":
        kw["topology"]["name"][0] = "C A"
    elif case == "resid":
        kw["topology"]["resid"][2] = -1
    elif case == "title":
        kw["title"] = "two\nlines"
    elif case == "time":
        kw["time"] = [0.0, np.nan]
    elif case == "step":
        kw["step"] = [0.5, 1]
    elif case == "chunk":
        kw["chunk_bytes"] = 0
    elif case == "shape":
        x = x[:, :2]
    fn = tmp_path / "w.gro"
    with pytest.raises(ValueError, match=match):
        gro.write_gro(str(fn), x, **kw)
    assert not fn.exists()


def test_reader_checks_before_the_device(tmp_path):
    from moleculekit_b200 import gro

    raw = og.write(frames(3, 2, 0), og.random_topology(3, 0), boxes(2))
    fn = tmp_path / "t.gro"
    fn.write_bytes(raw)
    with pytest.raises(ValueError, match="fields must name distinct blocks"):
        gro.read_gro_device(str(fn), fields=("x", "f"))
    with pytest.raises(ValueError, match="chunk_bytes must be positive"):
        gro.read_gro_device(str(fn), chunk_bytes=0)
    with pytest.raises(ValueError, match="scale must be finite"):
        gro.read_gro_device(str(fn), scale=float("inf"))
    with pytest.raises(ValueError, match="has no velocities"):
        gro.read_gro_device(str(fn), fields=("x", "v"))
    # inconsistent point spacing and a bad count line are frame-0 errors found on the host
    lines = raw.split(b"\n")
    lines[2] = lines[2][:20] + b"  1.000  2.00000  3.0" + lines[2][41:]
    fn.write_bytes(b"\n".join(lines))
    with pytest.raises(ValueError, match=r"frame 0, line 3, column 21: the decimal points of the first atom line are "
                                         r"not equally spaced"):
        gro.read_gro(str(fn))
    lines = raw.split(b"\n")
    lines[1] = b"three"
    fn.write_bytes(b"\n".join(lines))
    with pytest.raises(ValueError, match=r"frame 0, line 2, column 1: the atom count line b'three' does not start"):
        gro.read_gro(str(fn))
    fn.write_bytes(b" \n\n")
    with pytest.raises(ValueError, match="no frames"):
        gro.index_gro(str(fn))
