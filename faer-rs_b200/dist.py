"""Multi-GPU front end: 1-D block-column-cyclic layout helpers, the distributed LLT / LU entry points and the column-split GEMM.

One process per GPU (torchrun); `torch.distributed` is the plumbing (rendezvous, id exchange, status reduction); the
data path is the library's own NCCL broadcast of each factored panel (csrc/dist.cu), issued on a high-priority CUDA
stream so that it overlaps the trailing updates (look-ahead). The reference has no multi-process code
(SURVEY.md §2b); the layout follows SURVEY.md §8e: block column b (width nb) lives on rank b % P.

The layout helpers are pure index arithmetic (numpy / torch, CPU or GPU) and are unit-tested on CPU with a
world-size-2 gloo group (tests/test_dist_cpu.py).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi


# ---- layout (pure index arithmetic) ------------------------------------------------------------------
def num_blocks(n: int, nb: int) -> int:
    return (n + nb - 1) // nb


def owner_of_block(b: int, nranks: int) -> int:
    return b % nranks


def local_blocks(n: int, nb: int, nranks: int, rank: int) -> list[int]:
    """Global block-column indices owned by `rank`, in local storage order."""
    return list(range(rank, num_blocks(n, nb), nranks))


def local_cols(n: int, nb: int, nranks: int, rank: int) -> int:
    return sum(min(nb, n - b * nb) for b in local_blocks(n, nb, nranks, rank))


def local_col_offset(b: int, nb: int, nranks: int) -> int:
    """Local column offset of global block column b on its owner."""
    return (b // nranks) * nb


def global_col_indices(n: int, nb: int, nranks: int, rank: int) -> np.ndarray:
    """Global column index of every local column of `rank` (length local_cols)."""
    idx = [np.arange(b * nb, min(n, (b + 1) * nb)) for b in local_blocks(n, nb, nranks, rank)]
    return np.concatenate(idx) if idx else np.zeros(0, dtype=np.int64)


def scatter_block_cyclic(A, nb: int, nranks: int, rank: int):
    """Local part (n x local_cols, column-major for numpy inputs) of a replicated global matrix."""
    cols = global_col_indices(A.shape[0] if A.shape[0] == A.shape[1] else A.shape[1], nb, nranks, rank)
    if capi._is_torch(A):
        import torch
        return A[:, torch.as_tensor(cols, device=A.device)].T.contiguous().T
    return np.asfortranarray(A[:, cols])


def gather_block_cyclic(locals_, n: int, nb: int, nranks: int):
    """Inverse of scatter_block_cyclic: list of per-rank local matrices -> global n x n (numpy)."""
    out = np.zeros((locals_[0].shape[0], n), dtype=locals_[0].dtype, order="F")
    for r, loc in enumerate(locals_):
        out[:, global_col_indices(n, nb, nranks, r)] = loc
    return out


def column_slab(ncols: int, nranks: int, rank: int) -> tuple[int, int]:
    """[start, stop) of the contiguous column slab of `rank` in a 1-D column split of ncols columns over nranks ranks: widths
    differ by at most one, slabs ordered by rank (SURVEY.md 8e: GEMM shards by output columns, no reduction)."""
    base, extra = divmod(ncols, nranks)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


# ---- communicator ------------------------------------------------------------------------------------
def init_from_torch_distributed() -> None:
    """Create the library's NCCL communicator over the default torch.distributed group (collective call)."""
    import torch
    import torch.distributed as dist
    lib = capi.load()
    _bind(lib)
    rank, world = dist.get_rank(), dist.get_world_size()
    buf = (C.c_ubyte * 128)()
    if rank == 0:
        assert lib.faer_b200_dist_unique_id(buf) == 0
    t = torch.tensor(list(bytes(buf)), dtype=torch.uint8)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.broadcast(t, src=0)
    raw = bytes(t.cpu().tolist())
    buf2 = (C.c_ubyte * 128).from_buffer_copy(raw)
    assert lib.faer_b200_dist_init(rank, world, buf2) == 0


def finalize() -> None:
    lib = capi.load()
    _bind(lib)
    lib.faer_b200_dist_finalize()


_bound = False


def _bind(lib) -> None:
    global _bound
    if _bound:
        return
    lib.faer_b200_dist_unique_id.argtypes = [C.c_void_p]
    lib.faer_b200_dist_unique_id.restype = C.c_int
    lib.faer_b200_dist_init.argtypes = [C.c_int, C.c_int, C.c_void_p]
    lib.faer_b200_dist_init.restype = C.c_int
    lib.faer_b200_dist_finalize.argtypes = []
    lib.faer_b200_dist_finalize.restype = None
    lib.faer_b200_dist_llt_factor_in_place_f64.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                          capi.LltRegularization, C.c_int]
    lib.faer_b200_dist_llt_factor_in_place_f64.restype = capi.LltStatus
    lib.faer_b200_dist_partial_piv_lu_factor_in_place_f64.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t,
                                                                      C.c_void_p, C.c_void_p, C.c_int]
    lib.faer_b200_dist_partial_piv_lu_factor_in_place_f64.restype = C.c_size_t
    for suf in ("f64", "f32"):
        f = getattr(lib, f"faer_b200_dist_qr_factor_in_place_{suf}")
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_int]
        f.restype = C.c_longlong
    _bound = True


# ---- distributed LLT ---------------------------------------------------------------------------------
def cholesky_in_place(A_local, n: int, nb: int = 512, regularization=(0.0, 0.0), lookahead=True):
    """Distributed in-place LLT. `A_local`: torch CUDA tensor, column-major view (n x local_cols, stride (1, ld)).
    `lookahead`: bool, or the driver's bit mask (1 = look-ahead, 2 = purely local run, 4 = 512-wide leading blocks on
    one GPU, the schedule of the single-GPU entry point).
    Returns (fail_index or -1, regularisation count) reduced over the ranks of the default process group (if any)."""
    import torch
    lib = capi.load()
    _bind(lib)
    assert capi._is_torch(A_local) and A_local.is_cuda and A_local.dtype == torch.float64
    assert A_local.shape[0] == n and (A_local.shape[1] == 0 or A_local.stride(0) == 1)
    ld = A_local.stride(1) if A_local.shape[1] > 1 else max(n, 1)
    delta = C.c_double(float(regularization[0])); eps = C.c_double(float(regularization[1]))
    reg = capi.LltRegularization(C.cast(C.pointer(delta), C.c_void_p), C.cast(C.pointer(eps), C.c_void_p))
    st = lib.faer_b200_dist_llt_factor_in_place_f64(A_local.data_ptr(), ld, n, nb, reg,
                                                    int(lookahead) if not isinstance(lookahead, bool) else (1 if lookahead else 0))
    fail = int(st.value) if st.tag == 1 else -1
    cnt = int(st.value) if st.tag == 0 else 0
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            big = 1 << 62
            t = torch.tensor([fail if fail >= 0 else big, -cnt], dtype=torch.int64, device=A_local.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN)  # min failing index; counts are summed below
            c = torch.tensor([cnt], dtype=torch.int64, device=A_local.device)
            dist.all_reduce(c, op=dist.ReduceOp.SUM)
            fail = int(t[0].item()) if int(t[0].item()) < big else -1
            cnt = int(c.item())
    except ImportError:  # pragma: no cover
        pass
    return fail, cnt


# ---- distributed LU -----------------------------------------------------------------------------------
def lu_in_place(A_local, n: int, nb: int = 512, lookahead=True):
    """Distributed in-place P A = L U (square n x n). Returns (perm_fwd, perm_inv, transposition_count) as numpy int64
    arrays (identical on every rank); (P A)[i, :] = A[perm_fwd[i], :]. `lookahead`: bool, or the driver's bit mask
    (1 = look-ahead, 2 = purely local run that ignores an existing communicator; 3 = both)."""
    import torch
    lib = capi.load()
    _bind(lib)
    assert capi._is_torch(A_local) and A_local.is_cuda and A_local.dtype == torch.float64
    assert A_local.shape[0] == n and (A_local.shape[1] == 0 or A_local.stride(0) == 1)
    ld = A_local.stride(1) if A_local.shape[1] > 1 else max(n, 1)
    perm = np.zeros(n, dtype=np.int64); pinv = np.zeros(n, dtype=np.int64)
    cnt = lib.faer_b200_dist_partial_piv_lu_factor_in_place_f64(A_local.data_ptr(), ld, n, nb, perm.ctypes.data,
                                                                pinv.ctypes.data,
                                                                int(lookahead) if not isinstance(lookahead, bool) else (1 if lookahead else 0))
    return perm, pinv, int(cnt)


# ---- distributed QR -----------------------------------------------------------------------------------
def qr_in_place(A_local, nrows: int, ncols: int, block_size: int, local_only: bool = False):
    """Distributed in-place Householder QR without pivoting (nrows >= ncols; f64 or f32). `A_local`: torch CUDA tensor, column-major
    view (nrows x local_cols) of the block columns of width `block_size` owned by this rank. Returns Q_coeff (block_size x ncols
    CUDA tensor, column-major, identical on every rank). Raises RuntimeError on a rank-deficient block (the reference's column
    skipping crosses block boundaries: use linalg.qr_in_place on one GPU for such inputs)."""
    import torch
    lib = capi.load()
    _bind(lib)
    assert capi._is_torch(A_local) and A_local.is_cuda and A_local.dtype in (torch.float64, torch.float32)
    assert A_local.shape[0] == nrows and (A_local.shape[1] == 0 or A_local.stride(0) == 1) and nrows >= ncols
    ld = A_local.stride(1) if A_local.shape[1] > 1 else max(nrows, 1)
    H = torch.zeros((ncols, block_size), dtype=A_local.dtype, device=A_local.device).T  # column-major, ld = block_size
    suf = "f64" if A_local.dtype == torch.float64 else "f32"
    r = getattr(lib, f"faer_b200_dist_qr_factor_in_place_{suf}")(A_local.data_ptr(), ld, nrows, ncols, block_size, H.data_ptr(),
                                                                 2 if local_only else 0)
    if r < 0:
        raise RuntimeError("distributed QR met a rank-deficient block")
    return H


# ---- distributed GEMM: 1-D column split -----------------------------------------------------------------
def matmul(C_local, accum, A, B_local, alpha=1.0, src_rank=None, par=None) -> None:
    """C[:, slab] = [C[:, slab] +] alpha * A @ B[:, slab] on every rank, slab = column_slab(ncols, world, rank): the
    independent-output-tiles sharding of SURVEY.md 8e. `A` is replicated; `B_local` / `C_local` are this rank's column slabs.
    There is NO data-path collective in the product itself (each rank runs the single-GPU kernels on its slab; the k-order of
    every output element is the single-GPU one). If `src_rank` is given, `A` only holds valid data on that rank and is first
    broadcast over the default torch.distributed group (one NCCL broadcast, the only exchange)."""
    from . import linalg as la
    if src_rank is not None:
        import torch.distributed as td
        if td.is_available() and td.is_initialized() and td.get_world_size() > 1:
            assert capi._is_torch(A), "broadcasting A needs a torch tensor"
            # broadcast the storage as it is laid out (column-major views are transposes of contiguous tensors)
            buf = A if A.is_contiguous() else A.T
            assert buf.is_contiguous(), "A must be contiguous in row- or column-major order to be broadcast in place"
            td.broadcast(buf, src=src_rank)
    assert A.shape[0] == C_local.shape[0] and A.shape[1] == B_local.shape[0] and B_local.shape[1] == C_local.shape[1]
    if C_local.shape[1] == 0:
        return
    la.matmul(C_local, accum, A, B_local, alpha, par)
