"""K16 on degenerate quadruples in any orientation: collinear float32 points that are not axis-aligned give exactly
angle 0 and (sin, cos) = (0, 1) on the device, as in the float64 oracle; and the frame list must be int32."""
import numpy as np
import pytest

from oracle import dihedral_oracle as do

pytestmark = pytest.mark.gpu


def test_collinear_quadruples_on_device():
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda:0")
    K, F = 300, 40
    P = do.collinear_quads(K * F, 7).reshape(4, 3, F, K)         # quadruple k of frame f = P[:, :, f, k]
    X = np.ascontiguousarray(np.transpose(P, (3, 0, 1, 2)).reshape(4 * K, 3, F), dtype=np.float32)
    quads = np.arange(4 * K, dtype=np.int32).reshape(K, 4)
    d, q = torch.from_numpy(X).to(dev), torch.from_numpy(quads).to(dev)
    sc = dihedrals_device(d, q, True).cpu().numpy()
    ang = dihedrals_device(d, q, False).cpu().numpy()
    assert np.array_equal(ang, np.zeros((F, K), np.float32)) and not np.signbit(ang).any()
    assert np.array_equal(sc, np.tile(np.array([0.0, 1.0], np.float32), (F, K)))
    assert np.array_equal(do.project(X, quads, True), sc.astype(np.float64))
    assert np.array_equal(do.project(X, quads, False), ang.astype(np.float64))


def test_frames_must_be_int32():
    import torch
    from moleculekit_b200.dihedral import dihedrals_device

    dev = torch.device("cuda:0")
    X = torch.randn((8, 3, 5), device=dev)
    q = torch.arange(8, dtype=torch.int32, device=dev).reshape(2, 4)
    with pytest.raises(AssertionError):
        dihedrals_device(X, q, True, frames=torch.tensor([4, 1], device=dev))  # int64
    got = dihedrals_device(X, q, True, frames=torch.tensor([4, 1], dtype=torch.int32, device=dev))
    assert torch.equal(got, dihedrals_device(X, q, True)[[4, 1]])
