// The blocked Householder QR driver and the block-Householder sequences, written once over the complex-capable scalar kinds
// <R, CX> (c64 / c32 in cplx.cu, fx128 / cx128 in qr_dd.cu): the reference's recursion on the host with every product through
// gemm_t, every triangular solve through solve_lower_t and every sub-view through sub_t (tensor_ops.cuh). Only the unblocked leaf
// differs per kind: each including file defines qr_unblocked_t<R, CX> for its kinds before instantiating the driver.
// Views are in elements (COMPLEX units on an R* base for the complex kinds).
//
// Reference (faer/src/linalg):
//   qr/no_pivoting/factor.rs:137-256   qr_in_place_blocked: sub-blocks of block_size / 2 (1 when block_size <= QR_LEAF or
//                                      m * n < blocking_threshold), T blocks shifted into place and merged (190-226)
//   qr/no_pivoting/factor.rs:258-301   qr_in_place: columns >= rank of Q_coeff are zero with +inf on the block diagonals
//   householder.rs:132-272             upgrade_householder_factor: T = striu(V^H V), the diagonal (tau) kept
//   householder.rs:370-620             apply_block_householder_on_the_left
//   householder.rs:724-808             the sequences, forward and transposed
#pragma once
#include <algorithm>

#include "runtime.cuh"
#include "tensor_ops.cuh"

namespace fb {

constexpr int QR_LEAF = 16;

template <class R>
struct QrCtx {
  cudaStream_t st;
  int* d_row;
  R* tmp;  // block_size x ncols scratch of the block applies
  i64 blocking_threshold;
};

// qr_in_place_unblocked (factor.rs:11-86) on the view A from (row_start, col_start) over all of A's columns, tau of reflector
// `row` into Hrow[row] (a 1 x size view); returns the new row index. Defined by the file that instantiates the driver.
template <class R, bool CX>
i64 qr_unblocked_t(const QrCtx<R>& cx, View<R> A, View<R> Hrow, i64 row_start, i64 col_start);

namespace {

template <class R, bool CX>
__device__ __forceinline__ void qr_copy_el(R* p, i64 dst, i64 src) {
  if constexpr (CX) {
    const R re = p[2 * src], im = p[2 * src + 1];
    p[2 * dst] = re;
    p[2 * dst + 1] = im;
  } else {
    p[dst] = p[src];
  }
}

// factor.rs:190-203: after a leaf produced `local` reflectors with sub-block size sbs, the s2 x s2 upper-triangular T blocks
// sit in the first rows of H (view Hs: rows from `offset`, columns from `row`); block k moves down to rows [k, k + s2)
template <class R, bool CX>
__global__ void qr_shift_tblocks_kernel(R* __restrict__ Hs, i64 rs, i64 cs, int local, int sbs) {
  for (int e = threadIdx.x; e < local * sbs; e += blockDim.x) {
    const int col = e / sbs, i = e % sbs;
    const int k = (col / sbs) * sbs, j = col - k;
    if (k == 0 || i > j) continue;
    qr_copy_el<R, CX>(Hs, (i64)(k + i) * rs + (i64)col * cs, (i64)i * rs + (i64)col * cs);
  }
}

// factor.rs:283-299: columns >= rank of Q_coeff are zero with +inf on the block diagonals
template <class R, bool CX>
__global__ void qr_finish_kernel(R* __restrict__ H, i64 rs, i64 cs, int bs, int size, int rank) {
  const i64 e = (i64)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (i64)bs * (size - rank)) return;
  const int i = (int)(e % bs), j = rank + (int)(e / bs);
  const bool diag = i == j - (j / bs) * bs;
  R* p = H + (CX ? 2 : 1) * ((i64)i * rs + (i64)j * cs);
  p[0] = diag ? R(INFINITY) : R(0);
  if constexpr (CX) p[1] = R(0);
}

// upgrade_householder_factor (householder.rs:132-272): T = striu(V^H V), the diagonal (tau) kept
template <class R, bool CX>
void upgrade_householder_factor_t(cudaStream_t st, View<R> Tf, View<const R> V, i64 block_size, i64 prev_block_size) {
  if (block_size == prev_block_size || Tf.nrows <= prev_block_size) return;
  LaunchTag tag(LAUNCH_TBUILD);
  const i64 n = V.ncols;
  const i64 block_count = (Tf.nrows + block_size - 1) / block_size;
  if (block_count > 1) {
    const i64 mid = block_count / 2;  // householder.rs:155-157 splits at the block COUNT
    upgrade_householder_factor_t<R, CX>(st, sub_t<R, CX>(Tf, 0, 0, mid, mid), sub_t<R, CX>(V, 0, 0, V.nrows, mid), block_size,
                                        prev_block_size);
    upgrade_householder_factor_t<R, CX>(st, sub_t<R, CX>(Tf, mid, mid, Tf.nrows - mid, Tf.ncols - mid),
                                        sub_t<R, CX>(V, mid, mid, V.nrows - mid, V.ncols - mid), block_size, prev_block_size);
    return;
  }
  if (prev_block_size < 8) {
    View<const R> top = sub_t<R, CX>(V, 0, 0, n, n), bot = sub_t<R, CX>(V, n, 0, V.nrows - n, n);
    gemm_t<R, CX>(st, Tf, UNIT_UPPER, 0, top.t(), UNIT_UPPER, true, top, UNIT_LOWER, false, R(1));
    if (bot.nrows > 0) gemm_t<R, CX>(st, Tf, UNIT_UPPER, 1, bot.t(), RECT, true, bot, RECT, false, R(1));
  } else {
    const i64 prev_block_count = (Tf.nrows + prev_block_size - 1) / prev_block_size;
    const i64 mid = (prev_block_count / 2) * prev_block_size;
    View<R> tl = sub_t<R, CX>(Tf, 0, 0, mid, mid), tr = sub_t<R, CX>(Tf, 0, mid, mid, Tf.ncols - mid),
            br = sub_t<R, CX>(Tf, mid, mid, Tf.nrows - mid, Tf.ncols - mid);
    View<const R> left = sub_t<R, CX>(V, 0, 0, V.nrows, mid), right = sub_t<R, CX>(V, mid, mid, V.nrows - mid, V.ncols - mid);
    upgrade_householder_factor_t<R, CX>(st, tl, left, block_size, prev_block_size);
    upgrade_householder_factor_t<R, CX>(st, br, right, block_size, prev_block_size);
    View<const R> left2 = sub_t<R, CX>(left, mid, 0, left.nrows - mid, left.ncols);
    const i64 row_mid = right.ncols;
    View<const R> lt = sub_t<R, CX>(left2, 0, 0, row_mid, left2.ncols), lb = sub_t<R, CX>(left2, row_mid, 0, left2.nrows - row_mid, left2.ncols);
    View<const R> rt = sub_t<R, CX>(right, 0, 0, row_mid, right.ncols), rb = sub_t<R, CX>(right, row_mid, 0, right.nrows - row_mid, right.ncols);
    gemm_t<R, CX>(st, tr, RECT, 0, lt.t(), RECT, true, rt, UNIT_LOWER, false, R(1));
    if (lb.nrows > 0) gemm_t<R, CX>(st, tr, RECT, 1, lb.t(), RECT, true, rb, RECT, false, R(1));
  }
}

// apply_block_householder_on_the_left (householder.rs:370-620): M <- (I - V T^-1 V^H) M (forward = false) or
// (I - V T^-H V^H) M (forward = true), conj_lhs conjugating V and T; tmp: N x K scratch
template <class R, bool CX>
void apply_block_householder_left_t(cudaStream_t st, View<const R> V, View<const R> Tf, bool conj_lhs, View<R> M, bool forward, R* tmpbuf) {
  const i64 N = V.ncols, m = V.nrows, K = M.ncols;
  if (N == 0 || K == 0) return;
  LaunchTag tag(LAUNCH_PRODUCT);
  View<R> tmp{tmpbuf, N, K, 1, N};
  View<const R> Vt = sub_t<R, CX>(V, 0, 0, N, N), Vb = sub_t<R, CX>(V, N, 0, m - N, N);
  View<R> top = sub_t<R, CX>(M, 0, 0, N, K), bot = sub_t<R, CX>(M, N, 0, m - N, K);
  gemm_t<R, CX>(st, tmp, RECT, 0, Vt.t(), UNIT_UPPER, !conj_lhs, cview(top), RECT, false, R(1));
  if (m > N) gemm_t<R, CX>(st, tmp, RECT, 1, Vb.t(), RECT, !conj_lhs, cview(bot), RECT, false, R(1));
  if (forward) solve_lower_t<R, CX>(st, Tf.t(), false, !conj_lhs, tmp);
  else {
    // upper = lower on the views with rows and columns reversed
    View<const R> t{Tf.ptr + (CX ? 2 : 1) * ((N - 1) * Tf.rs + (N - 1) * Tf.cs), N, N, -Tf.rs, -Tf.cs};
    View<R> r{tmp.ptr + (CX ? 2 : 1) * ((N - 1) * tmp.rs), N, K, -tmp.rs, tmp.cs};
    solve_lower_t<R, CX>(st, t, false, conj_lhs, r);
  }
  gemm_t<R, CX>(st, top, RECT, 1, Vt, UNIT_LOWER, conj_lhs, cview(tmp), RECT, false, R(-1));
  if (m > N) gemm_t<R, CX>(st, bot, RECT, 1, Vb, RECT, conj_lhs, cview(tmp), RECT, false, R(-1));
}

// qr_in_place_blocked (factor.rs:137-256)
template <class R, bool CX>
i64 qr_blocked_t(const QrCtx<R>& cx, View<R> A, View<R> H, i64 row_start, i64 col_start) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n);
  const i64 block_size0 = H.nrows;
  if (block_size0 == 1) return qr_unblocked_t<R, CX>(cx, A, H, row_start, col_start);
  const i64 sub_block_size0 = (block_size0 <= QR_LEAF || m * n < cx.blocking_threshold) ? 1 : block_size0 / 2;
  i64 col = col_start, row = row_start;
  while (row < size && col < n) {
    const i64 block_size = std::min(block_size0, std::min(size - row, n - col));
    const i64 sub_block_size = std::min(block_size, sub_block_size0);
    const i64 start = row;
    i64 offset = 0;
    while (offset < block_size && col < n) {
      const i64 bsz = std::min(n - col, block_size - offset);
      const i64 sbs = std::min(bsz, sub_block_size);
      const i64 new_row = qr_blocked_t<R, CX>(cx, sub_t<R, CX>(A, 0, 0, m, col + bsz), sub_t<R, CX>(H, offset, 0, sbs, H.ncols), row, col);
      const i64 local = new_row - row;
      if (local > 0) {
        if (local > sbs) {
          View<R> Hs = sub_t<R, CX>(H, offset, row, H.nrows - offset, local);
          qr_shift_tblocks_kernel<R, CX><<<1, 256, 0, cx.st>>>(Hs.ptr, Hs.rs, Hs.cs, (int)local, (int)sbs);
          FB_CUDA_CHECK(cudaGetLastError());
          note_launch();
        }
        upgrade_householder_factor_t<R, CX>(cx.st, sub_t<R, CX>(H, offset, row, local, local), cview(sub_t<R, CX>(A, row, row, m - row, local)),
                                            local, sbs);
        if (offset > 0) {
          LaunchTag tag(LAUNCH_TBUILD);
          const i64 w = offset + local;
          View<R> Hh = sub_t<R, CX>(H, 0, start, w, w);
          View<const R> Aa = cview(sub_t<R, CX>(A, start, start, m - start, w));
          View<const R> A0 = sub_t<R, CX>(Aa, 0, 0, w, w), A1 = sub_t<R, CX>(Aa, w, 0, Aa.nrows - w, w);
          gemm_t<R, CX>(cx.st, Hh, UNIT_UPPER, 0, A0.t(), UNIT_UPPER, true, A0, UNIT_LOWER, false, R(1));
          if (A1.nrows > 0) gemm_t<R, CX>(cx.st, Hh, UNIT_UPPER, 1, A1.t(), RECT, true, A1, RECT, false, R(1));
        }
      }
      View<R> below = sub_t<R, CX>(A, row, 0, m - row, n);
      View<R> A1 = sub_t<R, CX>(below, 0, col + bsz, m - row, n - (col + bsz));
      if (A1.ncols > 0 && local > 0)
        apply_block_householder_left_t<R, CX>(cx.st, cview(sub_t<R, CX>(below, 0, row, m - row, local)),
                                              cview(sub_t<R, CX>(H, offset, row, local, local)), false, A1, true, cx.tmp);
      offset += local;
      row += local;
      col += bsz;
    }
  }
  return row;
}

// qr_in_place (factor.rs:258-301): returns the rank
template <class R, bool CX>
i64 qr_in_place_t(cudaStream_t st, View<R> A, View<R> Q_coeff, i64 blocking_threshold) {
  const i64 m = A.nrows, n = A.ncols, size = std::min(m, n), bs = Q_coeff.nrows;
  FB_ASSERT(bs > 0 && Q_coeff.ncols == size, "Q_coeff must be block_size x min(nrows, ncols)");
  if (size == 0) return 0;
  FB_ASSERT(m < (i64(1) << 31) && n < (i64(1) << 31), "complex QR dimensions limited to 2^31");
  int* d_row = (int*)ws_alloc(sizeof(int));
  R* tmp = (R*)ws_alloc((size_t)bs * (size_t)n * (CX ? 2 : 1) * sizeof(R));
  QrCtx<R> cx{st, d_row, tmp, blocking_threshold};
  const i64 rank = qr_blocked_t<R, CX>(cx, A, Q_coeff, 0, 0);
  if (rank < size) {
    const i64 cnt = bs * (size - rank);
    qr_finish_kernel<R, CX><<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(Q_coeff.ptr, Q_coeff.rs, Q_coeff.cs, (int)bs, (int)size, (int)rank);
    FB_CUDA_CHECK(cudaGetLastError());
    note_launch();
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(tmp);
  ws_free(d_row);
  return rank;
}

// apply_block_householder_sequence_[transpose_]on_the_left_in_place_with_conj (householder.rs:724-808): rhs <- Q rhs or Q^H rhs
// (with conj: the conjugated Q), Q given by its basis (unit-lower trapezoid) and block_size x size factor
template <class R, bool CX>
void apply_householder_sequence_left_t(cudaStream_t st, View<const R> basis, View<const R> factor, bool conj, View<R> rhs, bool transpose) {
  const i64 bs = factor.nrows, size = factor.ncols, m = basis.nrows, K = rhs.ncols;
  FB_ASSERT(bs > 0 && size == std::min(basis.nrows, basis.ncols) && rhs.nrows == m, "Householder sequence shape mismatch");
  if (size == 0 || K == 0) return;
  R* tmp = (R*)ws_alloc((size_t)bs * (size_t)K * (CX ? 2 : 1) * sizeof(R));
  if (transpose) {
    // householder.rs:768-808: blocks in ascending order, each through transpose_on_the_left = conj composed with Yes, forward
    for (i64 j = 0; j < size;) {
      const i64 b = std::min(bs, size - j);
      apply_block_householder_left_t<R, CX>(st, sub_t<R, CX>(basis, j, j, m - j, b), sub_t<R, CX>(factor, 0, j, b, b), !conj,
                                            sub_t<R, CX>(rhs, j, 0, m - j, K), true, tmp);
      j += b;
    }
  } else {
    // householder.rs:724-765: blocks in descending order (the last block may be short)
    i64 j = size, b = size % bs ? size % bs : bs;
    while (j > 0) {
      const i64 jp = j - b;
      apply_block_householder_left_t<R, CX>(st, sub_t<R, CX>(basis, jp, jp, m - jp, b), sub_t<R, CX>(factor, 0, jp, b, b), conj,
                                            sub_t<R, CX>(rhs, jp, 0, m - jp, K), false, tmp);
      j = jp;
      b = bs;
    }
  }
  FB_CUDA_CHECK(cudaStreamSynchronize(st));
  ws_free(tmp);
}

}  // namespace

}  // namespace fb
