"""The shared binding layer's argument checks, which run before any device work."""
import pytest


def test_index_arg():
    import torch
    from moleculekit_b200 import _lib

    cpu = torch.device("cpu")
    _lib.index_arg(None, cpu)
    _lib.index_arg(torch.arange(6, dtype=torch.int32), cpu)
    _lib.index_arg(torch.arange(8, dtype=torch.int32).reshape(2, 4), cpu, cols=4)
    _lib.index_arg(torch.arange(3), cpu, torch.int64)
    for bad, kw in ((torch.arange(6), {}),                                         # int64 where int32 is read
                    (torch.arange(12, dtype=torch.int32)[::2], {}),                # strided
                    (torch.arange(8, dtype=torch.int32).reshape(2, 4), {}),        # 2-D where 1-D is read
                    (torch.arange(8, dtype=torch.int32).reshape(4, 2), {"cols": 4}),
                    (torch.arange(6, dtype=torch.int32, device="meta"), {})):      # another device
        with pytest.raises(AssertionError):
            _lib.index_arg(bad, cpu, **kw)


def test_device_functions_refuse_cpu_tensors():
    import torch
    from moleculekit_b200 import _lib, align, coords

    X = torch.zeros((4, 3, 2))
    sel = torch.arange(4, dtype=torch.int32)
    for call in (lambda: align.superpose_device(X, sel, X, sel), lambda: align.rmsd_device(X, sel, X, sel),
                 lambda: align.apply_device(X, torch.zeros((2, align.RECORD), dtype=torch.float64)),
                 lambda: coords.coordinates_device(X, sel), lambda: coords.coord_sums_device(X, sel),
                 lambda: coords.fluctuation_device(X, sel, torch.zeros((4, 3), dtype=torch.float64))):
        with pytest.raises(_lib.MkbError, match="no CPU fallback"):
            call()
    with pytest.raises(_lib.MkbError, match="CUDA devices only"):
        _lib.device("cpu")
