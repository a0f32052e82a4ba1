"""Every writer checks a CUDA ``coords`` before it opens, and so creates or truncates, its file."""
import importlib

import pytest

from test_trajio_cpu import WRITERS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fmt", list(WRITERS))
def test_float64_cuda_coords_leave_an_existing_file_alone(tmp_path, fmt):
    import torch

    write = getattr(importlib.import_module(f"moleculekit_b200.{fmt}"), f"write_{fmt}")
    fn = tmp_path / f"precious.{fmt}"
    fn.write_bytes(b"precious")
    with pytest.raises(ValueError, match="coords must be float32"):
        write(str(fn), **dict(WRITERS[fmt], coords=torch.zeros((12, 3, 4), dtype=torch.float64, device="cuda")))
    assert fn.read_bytes() == b"precious"
