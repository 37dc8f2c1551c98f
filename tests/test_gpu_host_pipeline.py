"""GPU tests of the host-pointer LLT path (block columns streamed through the factorization, dist.cu LltHostPipe).

The pipeline runs the same right-looking block-column driver on the same kernels as the device-resident path, but in its first
step each trailing block column is updated by its own launch once its upload has landed, where the device-resident path
updates them all in one launch. The products are tiled differently and round differently in the last bit, hence the
assertion is 1e-13 relative, not bitwise. On top of that the reference's contract is
checked: the strict upper triangle of the host matrix is neither read nor written (cholesky/llt/factor.rs:68-97 reads the lower triangle only), and a non-positive pivot is reported with the
same index (ldlt/factor.rs:146-150)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _spd(n, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, 64))
    A = G @ G.T + n * np.eye(n)
    return np.asfortranarray(A)


@pytest.mark.parametrize("n", [4096, 5000])
def test_host_llt_equals_device_llt(fb, cuda_dev, n):
    import torch
    la = fb.linalg
    A = _spd(n, 11)
    dA = torch.from_numpy(A).to(cuda_dev).T.contiguous().T  # column-major device copy
    la.cholesky_in_place(dA)
    want = np.tril(dA.cpu().numpy())
    host = A.copy(order="F")
    host[np.triu_indices(n, 1)] = np.nan  # must never be read
    info = la.cholesky_in_place(host)
    assert info.dynamic_regularization_count == 0
    assert np.all(np.isnan(host[np.triu_indices(n, 1)]))
    assert np.abs(np.tril(host) - want).max() <= 1e-13 * np.abs(want).max()
    # and it is a Cholesky factor
    L = np.tril(host)
    x = np.random.default_rng(1).standard_normal((n, 2))
    assert np.abs(A @ x - L @ (L.T @ x)).max() <= 1e-10 * np.abs(A).max() * n


@pytest.mark.parametrize("bad", [1000, 3001])  # an early and a later block column
def test_host_llt_reports_the_failing_column(fb, bad):
    la = fb.linalg
    n = 4200
    A = _spd(n, 12)
    A[bad, bad] = -1.0
    with pytest.raises(la.LltError) as e:
        la.cholesky_in_place(A)
    assert e.value.index == bad
