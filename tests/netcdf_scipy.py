"""TEST INFRASTRUCTURE: AMBER NetCDF files written and read by scipy.io.netcdf_file, an implementation of netCDF-3
independent of moleculekit_b200.netcdf.  It keeps float32 bit patterns (NaN payloads, signalling NaNs, -0.0) as they
are in both directions."""
import io

import numpy as np
from scipy.io import netcdf_file


def amber_file(x, box=None, angles=None, time=None, title="written by moleculekit_b200", version=2, extras=False,
               program="moleculekit_b200", program_version=None) -> bytes:
    """The AMBER convention 1.0 trajectory of coordinates ``x`` (F, N, 3) float32 as scipy writes it.  ``box`` /
    ``angles`` (F, 3) add cell_lengths / cell_angles (angles 90 when only ``box`` is given); ``time`` (F,) defaults to
    the frame index.  ``extras`` adds velocities, forces, a 2-int remd_indices and a 3-byte record variable before
    coordinates, so coordinates is not first in the record and a padded slab precedes it."""
    if program_version is None:
        from moleculekit_b200 import __version__ as program_version
    x = np.asarray(x, np.float32)
    F, N, _ = x.shape
    fh = io.BytesIO()
    f = netcdf_file(fh, "w", version=version)
    f.title = title
    f.application = "moleculekit_b200"
    f.program = program
    f.programVersion = program_version
    f.Conventions = "AMBER"
    f.ConventionVersion = "1.0"
    f.createDimension("frame", None)
    f.createDimension("spatial", 3)
    f.createDimension("atom", N)
    if box is not None:
        f.createDimension("cell_spatial", 3)
        f.createDimension("label", 5)
        f.createDimension("cell_angular", 3)
    if extras:
        f.createDimension("remd_dimension", 2)
        f.createDimension("odd", 3)
    v = f.createVariable("spatial", "c", ("spatial",))
    v[:] = np.array(list("xyz"), "S1")
    v = f.createVariable("time", "f", ("frame",))
    v.units = "picosecond"
    v[:] = np.arange(F, dtype=np.float32) if time is None else np.asarray(time, np.float32)
    if extras:
        rng = np.random.default_rng(F + N)
        for name in ("velocities", "forces"):
            v = f.createVariable(name, "f", ("frame", "atom", "spatial"))
            v[:] = rng.normal(size=(F, N, 3)).astype(np.float32)
        v = f.createVariable("remd_indices", "i", ("frame", "remd_dimension"))
        v[:] = rng.integers(0, 9, size=(F, 2)).astype(np.int32)
        v = f.createVariable("odd_bytes", "b", ("frame", "odd"))
        v[:] = rng.integers(-9, 9, size=(F, 3)).astype(np.int8)
    v = f.createVariable("coordinates", "f", ("frame", "atom", "spatial"))
    v.units = "angstrom"
    v[:] = x
    if box is not None:
        v = f.createVariable("cell_spatial", "c", ("cell_spatial",))
        v[:] = np.array(list("abc"), "S1")
        v = f.createVariable("cell_angular", "c", ("cell_angular", "label"))
        v[:] = np.array([list("alpha"), list("beta "), list("gamma")], "S1")
        v = f.createVariable("cell_lengths", "d", ("frame", "cell_spatial"))
        v.units = "angstrom"
        v[:] = np.asarray(box, np.float64)
        v = f.createVariable("cell_angles", "d", ("frame", "cell_angular"))
        v.units = "degree"
        v[:] = np.full((F, 3), 90.0) if angles is None else np.asarray(angles, np.float64)
    f.flush()
    raw = fh.getvalue()
    f.fp = io.BytesIO()  # close() flushes once more: let it write elsewhere
    f.close()
    return raw


def read(raw: bytes) -> dict:
    """scipy's view of a file: its variables (copied), numrecs and recsize"""
    f = netcdf_file(io.BytesIO(raw), "r", mmap=False)
    out = dict(variables={k: np.array(v.data) for k, v in f.variables.items()}, numrecs=f._recs, recsize=f._recsize,
               version=int(f.version_byte), attributes=dict(f._attributes))
    f.close()
    return out
