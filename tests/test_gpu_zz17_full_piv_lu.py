"""Full-pivoting LU (`full_piv_lu_*`, csrc/full_piv_lu.cu) through the C ABI against the numpy restatement of
faer/src/linalg/lu/full_pivoting (tests/full_piv_lu_model.py).

Factor: row / column perm_fwd, perm_bwd and the transposition count exact, LU within tolerance, on inputs whose pivot sequence the
model gives the same in the working precision and in a wider one (the test checks that itself). Ties: integer inputs whose
elimination is exact in binary, so every tie is a real tie, follow the first-maximum rule exactly. Large Gaussian inputs: the
factor reproduces A, the multipliers are bounded, U's rows are dominated by their diagonal and runs are bitwise reproducible.
Solves, reconstruct and inverse per dtype and index width, and solvers.FullPivLu end to end."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import full_piv_lu_model as M  # noqa: E402

pytestmark = pytest.mark.gpu
DTYPES = [np.float64, np.float32, np.complex128, np.complex64]
WIDER = {np.float64: np.longdouble, np.float32: np.float64, np.complex128: np.clongdouble, np.complex64: np.complex128}
ITS = {"u32": np.uint32, "u64": np.uint64}
TORCH_IT = {"u32": "int32", "u64": "int64"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ueps(dtype):
    return float(np.finfo(dtype).eps)


def randn(rng, shape, dtype):
    x = rng.standard_normal(shape)
    if np.issubdtype(dtype, np.complexfloating):
        x = x + 1j * rng.standard_normal(shape)
    return np.asfortranarray(x.astype(dtype))


def strides_of(A):
    return A.strides[0] // A.itemsize, A.strides[1] // A.itemsize


def model(A):
    """The model's factor of A as the C ABI sees it (the branch from A's strides)."""
    rs, cs = strides_of(A)
    X = np.array(A, copy=True)
    rf, rb, cf, cb, cnt = M.lu_in_place(X, row_major=M.takes_transposed_branch(rs, cs))
    return X, rf, rb, cf, cb, cnt


def model_wider(A):
    rs, cs = strides_of(A)
    X = np.array(A, dtype=WIDER[A.dtype.type], copy=True)
    return M.lu_in_place(X, row_major=M.takes_transposed_branch(rs, cs))


def stable_pivots(A):
    w = model(A)
    x = model_wider(A)
    return all(np.array_equal(a, b) for a, b in zip(w[1:5], x[0:4])) and w[5] == x[4]


def gpu_factor(fb, A, it, device=False):
    """The library's factor of A (host array, or a CUDA tensor with the same strides when `device`)."""
    m, n = A.shape
    if device:
        import torch
        dt = getattr(torch, TORCH_IT[it])
        t = torch.from_numpy(np.array(A, copy=True)).cuda()
        if A.flags.f_contiguous and not A.flags.c_contiguous:
            t = torch.from_numpy(np.ascontiguousarray(A.T)).cuda().T
        rf, rb = torch.zeros(m, dtype=dt, device="cuda"), torch.zeros(m, dtype=dt, device="cuda")
        cf, cb = torch.zeros(n, dtype=dt, device="cuda"), torch.zeros(n, dtype=dt, device="cuda")
        info = fb.linalg.full_piv_lu_in_place(t, rf, rb, cf, cb)
        return (t.cpu().numpy(), rf.cpu().numpy().astype(np.int64), rb.cpu().numpy().astype(np.int64),
                cf.cpu().numpy().astype(np.int64), cb.cpu().numpy().astype(np.int64), info.transposition_count)
    X = A.copy(order="K")
    rf, rb = np.zeros(m, ITS[it]), np.zeros(m, ITS[it])
    cf, cb = np.zeros(n, ITS[it]), np.zeros(n, ITS[it])
    info = fb.linalg.full_piv_lu_in_place(X, rf, rb, cf, cb)
    return X, rf.astype(np.int64), rb.astype(np.int64), cf.astype(np.int64), cb.astype(np.int64), info.transposition_count


def check_against_model(got, want, dtype):
    X, rf, rb, cf, cb, cnt = got
    Xm, rfm, rbm, cfm, cbm, cntm = want
    assert np.array_equal(rf, rfm) and np.array_equal(rb, rbm)
    assert np.array_equal(cf, cfm) and np.array_equal(cb, cbm)
    assert cnt == cntm
    m, n = X.shape
    if X.size:
        scale = max(1.0, float(np.max(np.abs(Xm))))
        assert np.max(np.abs(X.astype(np.complex128) - Xm.astype(np.complex128))) <= 40 * max(m, n) * ueps(dtype) * scale


def stable_input(shape, dtype, seed0):
    for seed in range(seed0, seed0 + 6):
        A = randn(np.random.default_rng(seed), shape, dtype)
        if stable_pivots(A):
            return A
    raise AssertionError(f"no input of shape {shape} with rounding-independent pivots")


_CACHE = {}


def stable_case(shape, dtype):
    key = (shape, np.dtype(dtype).name)
    if key not in _CACHE:
        A = stable_input(shape, dtype, 1000 * shape[0] + shape[1])
        _CACHE[key] = (A, model(A))
    return _CACHE[key]


SHAPES = [(0, 0), (0, 5), (1, 1), (2, 2), (3, 3), (17, 17), (127, 127), (255, 255), (1000, 1000), (2000, 300), (300, 2000),
          (1, 9), (9, 1)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("it", ["u32", "u64"])
@pytest.mark.parametrize("shape", SHAPES)
def test_factor_matches_model(fb, dtype, it, shape):
    if shape[0] == 0 or shape[1] == 0:
        A = np.zeros(shape, dtype=dtype, order="F")
        want = model(A)
    else:
        A, want = stable_case(shape, dtype)
    check_against_model(gpu_factor(fb, A, it), want, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(17, 17), (255, 255), (300, 200)])
def test_factor_device_pointers(fb, cuda_dev, dtype, shape):
    A, want = stable_case(shape, dtype)
    for it in ("u32", "u64"):
        check_against_model(gpu_factor(fb, A, it, device=True), want, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(40, 40), (255, 255), (120, 70), (70, 120)])
def test_factor_row_major_takes_the_transposed_branch(fb, dtype, shape):
    for seed in range(6):
        A = np.ascontiguousarray(randn(np.random.default_rng(seed), shape, dtype))
        if stable_pivots(A):
            break
    else:
        raise AssertionError("no stable row-major input")
    assert M.takes_transposed_branch(*strides_of(A))
    check_against_model(gpu_factor(fb, A, "u64"), model(A), dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_factor_strided_view(fb, dtype):
    for seed in range(6):
        big = randn(np.random.default_rng(seed), (2 * 150, 3 * 90), dtype)
        A = big[::2, ::3]  # row stride 2: through the compact copy
        if stable_pivots(A):
            break
    else:
        raise AssertionError("no stable strided input")
    want = model(A)
    rf, rb, cf, cb = (np.zeros(k, np.uint64) for k in (150, 150, 90, 90))
    view = big.copy(order="F")
    sub = view[::2, ::3]
    info = fb.linalg.full_piv_lu_in_place(sub, rf, rb, cf, cb)
    check_against_model((np.array(sub), rf.astype(np.int64), rb.astype(np.int64), cf.astype(np.int64), cb.astype(np.int64),
                         info.transposition_count), want, dtype)
    untouched = np.ones(view.shape, bool)
    untouched[::2, ::3] = False
    assert np.array_equal(view[untouched], big[untouched])


# ---- ties ----
def exact_tie_inputs(dtype, count=4):
    """Small integer matrices with many equal entries whose elimination is exact in binary: the model's factor is identical in the
    working precision and in the wider one (so no tie is a rounding artefact)."""
    out = []
    rng = np.random.default_rng(7)
    tries = 0
    while len(out) < count and tries < 2000:
        tries += 1
        m, n = int(rng.integers(3, 14)), int(rng.integers(3, 14))
        A = rng.choice([-2.0, -1.0, 0.0, 0.0, 1.0, 2.0], size=(m, n))
        if np.issubdtype(dtype, np.complexfloating):
            A = A + 1j * rng.choice([-1.0, 0.0, 0.0, 1.0], size=(m, n))
        A = np.asfortranarray(A.astype(dtype))
        w = model(A)
        x = model_wider(A)
        if not all(np.array_equal(a, b) for a, b in zip(w[1:5], x[0:4])):
            continue
        Xw = np.array(A, dtype=WIDER[dtype], copy=True)
        M.lu_in_place(Xw)
        if not np.array_equal(np.array(w[0], dtype=WIDER[dtype]), Xw):
            continue
        # many exact ties in the first search
        s = M.abs1(A)
        if np.count_nonzero(s == s.max()) < 2:
            continue
        out.append(A)
    assert len(out) == count
    return out


@pytest.mark.parametrize("dtype", DTYPES)
def test_exact_ties_follow_the_first_maximum_rule(fb, dtype):
    for A in exact_tie_inputs(dtype):
        want = model(A)
        got = gpu_factor(fb, A, "u64")
        check_against_model(got, want, dtype)
        assert np.array_equal(got[0], want[0])  # no rounding anywhere: the factor is exact


def test_gh238_factor_and_solve_are_finite(fb):
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "full_piv_lu_gh238.json")))
    n = d["n"]
    A = np.asfortranarray(np.array(d["A_row_major"]).reshape(n, n))
    b = np.array(d["b"]).reshape(n, 1)
    lu = fb.solvers.full_piv_lu(A)
    assert np.all(np.isfinite(lu.L())) and np.all(np.isfinite(lu.U()))
    x = lu.solve(b)
    assert np.all(np.isfinite(x))
    want = model(A)
    got = gpu_factor(fb, A, "u64")
    check_against_model(got, want, np.float64)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["zero", "ones", "identity"])
def test_structured_inputs(fb, dtype, kind):
    for shape in [(6, 6), (7, 4), (4, 7)]:
        A = {"zero": np.zeros(shape), "ones": np.ones(shape), "identity": np.eye(*shape)}[kind]
        A = np.asfortranarray(A.astype(dtype))
        got = gpu_factor(fb, A, "u32")
        want = model(A)
        check_against_model(got, want, dtype)
        assert np.array_equal(got[0], want[0])
        assert got[5] == 0
        if kind == "zero":
            assert np.array_equal(got[0], A)


# ---- large ----
@pytest.mark.parametrize("dtype,n", [(np.float64, 4096), (np.complex64, 2048)])
def test_large_gaussian(fb, cuda_dev, dtype, n):
    import torch
    rng = np.random.default_rng(11)
    A = randn(rng, (n, n), dtype)
    tA = torch.from_numpy(np.ascontiguousarray(A.T)).cuda().T

    def factor():
        X = tA.clone().T.contiguous().T
        ps = [torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(4)]
        info = fb.linalg.full_piv_lu_in_place(X, *ps)
        return X, ps, info.transposition_count

    X1, ps1, c1 = factor()
    X2, ps2, c2 = factor()
    assert torch.equal(X1, X2) and c1 == c2
    assert all(torch.equal(a, b) for a, b in zip(ps1, ps2))
    L = torch.tril(X1, -1) + torch.eye(n, dtype=X1.dtype, device="cuda")
    U = torch.triu(X1)
    L = L.T.contiguous().T
    U = U.T.contiguous().T
    out = torch.zeros((n, n), dtype=X1.dtype, device="cuda").T
    fb.linalg.full_piv_lu_reconstruct(out, L, U, *ps1)
    err = (out - tA).abs().max().item()
    assert err <= 50 * n * ueps(dtype) * tA.abs().max().item(), err
    a1 = (lambda z: z.real.abs() + z.imag.abs()) if X1.is_complex() else (lambda z: z.abs())
    lbound = (np.sqrt(2.0) if X1.is_complex() else 1.0) * (1 + 8 * ueps(dtype))
    assert torch.tril(X1, -1).abs().max().item() <= lbound
    d = a1(torch.diagonal(U))
    assert torch.all(a1(torch.triu(U, 1)) <= d[:, None])


# ---- solves and products ----
def factors(fb, A, it):
    X, rf, rb, cf, cb, _ = gpu_factor(fb, A, it)
    L, U = M.split(X)
    cast = ITS[it]
    return np.asfortranarray(L), np.asfortranarray(U), [p.astype(cast) for p in (rf, rb, cf, cb)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("it", ["u32", "u64"])
def test_solves(fb, dtype, it):
    rng = np.random.default_rng(3)
    n, k = 50, 3
    A = randn(rng, (n, n), dtype)
    B = randn(rng, (n, k), dtype)
    L, U, ps = factors(fb, A, it)
    tol = 200 * n * ueps(dtype) * np.linalg.cond(A.astype(np.complex128))
    for conj in (0, 1):
        Ac = np.conj(A) if conj else A
        X = B.copy(order="F")
        fb.linalg.full_piv_lu_solve_in_place(L, U, *ps, X, conj)
        assert np.max(np.abs(Ac @ X - B)) <= tol * np.max(np.abs(B))
        X = B.copy(order="F")
        fb.linalg.full_piv_lu_solve_transpose_in_place(L, U, *ps, X, conj)
        assert np.max(np.abs(Ac.T @ X - B)) <= tol * np.max(np.abs(B))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("it", ["u32", "u64"])
@pytest.mark.parametrize("shape", [(50, 50), (100, 50), (50, 100)])
def test_reconstruct(fb, dtype, it, shape):
    A = randn(np.random.default_rng(5), shape, dtype)
    L, U, ps = factors(fb, A, it)
    out = np.zeros(shape, dtype=dtype, order="F")
    fb.linalg.full_piv_lu_reconstruct(out, L, U, *ps)
    assert np.max(np.abs(out - A)) <= 50 * max(shape) * ueps(dtype) * np.max(np.abs(A))
    want = M.reconstruct(L, U, ps[1].astype(np.int64), ps[3].astype(np.int64))
    assert np.max(np.abs(out - want)) <= 50 * max(shape) * ueps(dtype) * np.max(np.abs(A))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("it", ["u32", "u64"])
def test_inverse(fb, dtype, it):
    n = 50
    A = randn(np.random.default_rng(6), (n, n), dtype)
    L, U, ps = factors(fb, A, it)
    out = np.zeros((n, n), dtype=dtype, order="F")
    fb.linalg.full_piv_lu_inverse(out, L, U, *ps)
    tol = 200 * n * ueps(dtype) * np.linalg.cond(A.astype(np.complex128))
    assert np.max(np.abs(out @ A - np.eye(n))) <= tol
    want = M.inverse(L.astype(np.complex128), U.astype(np.complex128), ps[1].astype(np.int64), ps[3].astype(np.int64))
    assert np.max(np.abs(out - want)) <= tol * np.max(np.abs(want))


# ---- solver ----
@pytest.mark.parametrize("dtype", DTYPES)
def test_solver_numpy_and_torch(fb, cuda_dev, dtype):
    import torch
    rng = np.random.default_rng(9)
    n = 60
    A = randn(rng, (n, n), dtype)
    b = randn(rng, (n, 2), dtype)
    tol = 200 * n * ueps(dtype) * np.linalg.cond(A.astype(np.complex128)) * np.max(np.abs(b))
    lu = fb.solvers.full_piv_lu(A)
    assert lu.nrows() == n and lu.ncols() == n
    pf, pb = lu.P()
    qf, qb = lu.Q()
    PAQ = A[np.ix_(pf.astype(np.int64), qf.astype(np.int64))]
    assert np.max(np.abs(lu.L() @ lu.U() - PAQ)) <= 50 * n * ueps(dtype) * np.max(np.abs(A))
    assert np.max(np.abs(A @ lu.solve(b) - b)) <= tol
    assert np.max(np.abs(A.T @ lu.solve_transpose(b) - b)) <= tol
    assert np.max(np.abs(np.conj(A) @ lu.solve_conjugate(b) - b)) <= tol
    assert np.max(np.abs(np.conj(A).T @ lu.solve_adjoint(b) - b)) <= tol
    assert np.max(np.abs(lu.reconstruct() - A)) <= 50 * n * ueps(dtype) * np.max(np.abs(A))
    assert np.max(np.abs(lu.inverse() @ A - np.eye(n))) <= tol / np.max(np.abs(b))
    tA = torch.from_numpy(np.ascontiguousarray(A.T)).cuda().T
    tb = torch.from_numpy(np.ascontiguousarray(b.T)).cuda().T
    tlu = fb.solvers.full_piv_lu(tA)
    x = tlu.solve(tb).cpu().numpy()
    assert np.max(np.abs(A @ x - b)) <= tol
    assert np.max(np.abs(tlu.reconstruct().cpu().numpy() - A)) <= 50 * n * ueps(dtype) * np.max(np.abs(A))
    for r in (60, 40):
        R = randn(rng, (r, 100 - r), dtype)
        rlu = fb.solvers.full_piv_lu(R)
        assert np.max(np.abs(rlu.reconstruct() - R)) <= 50 * 100 * ueps(dtype) * np.max(np.abs(R))
