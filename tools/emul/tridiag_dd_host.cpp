// Host run of the double-double (fx128) real tridiagonal eigensolvers of csrc/evd_dd.cu: the SAME scalar routines the GPU kernels
// call (tridiag_dc_core.cuh and tridiag_ev.cuh through their dd instantiation, tridiag_dd.cuh) with the kernels' glue written as
// plain loops in the same order of operations: power-of-two scaling, tears, one-thread QL leaves, merge order by ranks, deflation
// scan, secular roots, Gu-Eisenstat z-hat, vectors, Givens folding, output ordering, Q_new = Q_old W; and the Gershgorin interval
// plus one bisection per value. Also a dd evaluation of the residual and of U^T U - I. Test infrastructure for
// tests/test_tridiag_dd_host_cpu.py, not product code. Build with -ffp-contract=off (dd.cuh's host arithmetic must not be fused).
//
// -DTDD_SLOPPY builds the negative control: dc_sub<dd> is faer's own subtraction add(a, -b) instead of dd_sub_accurate.
#include <algorithm>
#include <cmath>
#include <vector>

#ifdef TDD_SLOPPY
#include "../../faer-rs_b200/csrc/dd.cuh"
#include "../../faer-rs_b200/csrc/tridiag_dc_core.cuh"
#include "../../faer-rs_b200/csrc/tridiag_ev.cuh"
namespace fb {
namespace dc {
template <>
struct DcLim<dd> {
  static dd eps() { return dd_eps(); }
  static dd tiny() { return dd_min_positive(); }
};
template <>
dd dc_sub<dd>(dd a, dd b) {
  return a - b;
}
}  // namespace dc
namespace tev {
template <>
struct Lim<dd> {
  static dd eps() { return dd_eps(); }
  static dd safmin() { return dd_min_positive(); }
};
}  // namespace tev
}  // namespace fb
#else
#include "../../faer-rs_b200/csrc/tridiag_dd.cuh"
#endif

using fb::dd;

namespace {
const int LEAF = 32;
struct Merge {
  int lo, mid, hi;
};
int num_levels(long long n) {
  int lv = 0;
  while (((n + (1ll << lv) - 1) >> lv) > LEAF) ++lv;
  return lv;
}
std::vector<dd> load(const double* hi, const double* lo, int n) {
  std::vector<dd> v((size_t)std::max(n, 1), dd(0.0));
  for (int i = 0; i < n; ++i) v[(size_t)i] = dd(hi[i], lo[i]);
  return v;
}
int count_less(const dd* a, int n, dd x, bool or_equal) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (or_equal ? (a[mid] <= x) : (a[mid] < x)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
}  // namespace

// eigenvalues (ascending) by bisection, one per value (evd_dd.cu: ed_bounds_kernel, ed_values_kernel)
extern "C" void tdd_values(const double* dh, const double* dl_, const double* eh, const double* el, int n, double* oh, double* ol) {
  using namespace fb;
  const std::vector<dd> d = load(dh, dl_, n), e = load(eh, el, n - 1);
  dd lo = d[0], hi = d[0], e2(0.0);
  for (int i = 0; i < n; ++i) {
    const dd r = (i > 0 ? fabs(e[i - 1]) : dd(0.0)) + (i + 1 < n ? fabs(e[i]) : dd(0.0));
    lo = fmin(lo, d[i] - r);
    hi = fmax(hi, d[i] + r);
    if (i + 1 < n) e2 = fmax(e2, e[i] * e[i]);
  }
  const dd span = fmax(fabs(lo), fabs(hi));
  const dd pad = dd(4.0) * dd_eps() * span * dd((double)n) + dd_min_positive();
  for (int k = 0; k < n; ++k) {
    const dd v = tev::st_kth_smallest<dd>(d.data(), e.data(), n, k, lo - pad, hi + pad, e2);
    oh[k] = v.hi;
    ol[k] = v.lo;
  }
}

// eigenvalues (ascending) and eigenvectors (n x n column-major) by divide and conquer (evd_dd.cu: tridiag_dc_dd); 0 on success
extern "C" int tdd_eig(const double* dh, const double* dl_, const double* eh, const double* el, int n, double* lh, double* ll,
                       double* qh, double* ql) {
  using namespace fb;
  std::vector<dd> d = load(dh, dl_, n), e(n, dd(0.0));
  for (int i = 0; i + 1 < n; ++i) e[i] = dd(eh[i], el[i]);
  double mx = 0.0;
  for (int i = 0; i < n; ++i) mx = std::fmax(mx, std::fmax(std::fabs(d[i].hi), i + 1 < n ? std::fabs(e[i].hi) : 0.0));
  int ex = 0;
  if (mx > 0.0) std::frexp(mx, &ex);
  const dd s(std::ldexp(1.0, ex)), si(std::ldexp(1.0, -ex));
  for (int i = 0; i < n; ++i) {
    d[i] = d[i] * si;
    e[i] = i + 1 < n ? e[i] * si : dd(0.0);
  }
  const int nlev = num_levels(n);
  std::vector<std::vector<Merge>> levels((size_t)nlev);
  for (int l = 0; l < nlev; ++l)
    for (long long i = 0; i < (1ll << l); ++i)
      levels[(size_t)l].push_back({(int)((i * n) >> l), (int)(((2 * i + 1) * n) >> (l + 1)), (int)(((i + 1) * n) >> l)});
  std::vector<std::vector<dd>> rho((size_t)nlev), sgn((size_t)nlev);
  for (int l = 0; l < nlev; ++l)
    for (const Merge& m : levels[(size_t)l]) {
      const dd beta = e[m.mid - 1];
      rho[(size_t)l].push_back(fabs(beta));
      sgn[(size_t)l].push_back(beta < dd(0.0) ? dd(-1.0) : dd(1.0));
      d[m.mid - 1] = d[m.mid - 1] - fabs(beta);
      d[m.mid] = d[m.mid] - fabs(beta);
    }
  const size_t nn = (size_t)n * n;
  std::vector<dd> Qa(nn, dd(0.0)), Qb(nn, dd(0.0)), W(nn), DEL(nn);
  for (long long leaf = 0; leaf < (1ll << nlev); ++leaf) {
    const int lo = (int)((leaf * n) >> nlev), sz = (int)(((leaf + 1) * n) >> nlev) - lo;
    dd sd[LEAF], se[LEAF], Z[LEAF][LEAF + 1];
    for (int i = 0; i < LEAF; ++i) {
      sd[i] = i < sz ? d[lo + i] : dd(0.0);
      se[i] = i + 1 < sz ? e[lo + i] : dd(0.0);
      for (int j = 0; j < LEAF; ++j) Z[i][j] = dd(i == j ? 1.0 : 0.0);
    }
    const bool ok = dc::ql_implicit(sd, se, sz, [&](int i, dd c, dd sn) {
      for (int r = 0; r < sz; ++r) {
        const dd f = Z[r][i + 1];
        Z[r][i + 1] = sn * Z[r][i] + c * f;
        Z[r][i] = c * Z[r][i] - sn * f;
      }
    });
    if (!ok) return -2;
    for (int i = 0; i < sz; ++i) {
      int kmin = i;
      for (int j = i + 1; j < sz; ++j)
        if (sd[j] < sd[kmin]) kmin = j;
      if (kmin != i) {
        std::swap(sd[i], sd[kmin]);
        for (int r = 0; r < sz; ++r) std::swap(Z[r][i], Z[r][kmin]);
      }
    }
    for (int i = 0; i < sz; ++i) d[lo + i] = sd[i];
    for (int c = 0; c < sz; ++c)
      for (int r = 0; r < sz; ++r) Qa[(size_t)(lo + c) * n + lo + r] = Z[r][c];
  }
  std::vector<dd> dsort(n), zsort(n), dlv(n), w(n), ddf(n), rc(n), rs(n), lam(n), zh(n), dnew(n);
  std::vector<int> colsort(n), cnd(n), cdf(n), ra(n), rb(n), outcol(n);
  dd* cur = Qa.data();
  dd* nxt = Qb.data();
  const dd r2 = sqrt(dd(0.5));
  for (int l = nlev - 1; l >= 0; --l) {
    std::fill(W.begin(), W.end(), dd(0.0));
    for (size_t mi = 0; mi < levels[(size_t)l].size(); ++mi) {
      const Merge m = levels[(size_t)l][mi];
      const int lo = m.lo, mid = m.mid, hi = m.hi, sz = hi - lo;
      // prepare
      for (int i = lo; i < hi; ++i) {
        const dd zi = (i < mid ? cur[(size_t)i * n + (mid - 1)] : sgn[(size_t)l][mi] * cur[(size_t)i * n + mid]) * r2;
        const dd di = d[i];
        const int pos = i < mid ? (i - lo) + count_less(d.data() + mid, hi - mid, di, false)
                                : (i - mid) + count_less(d.data() + lo, mid - lo, di, true);
        dsort[lo + pos] = di;
        zsort[lo + pos] = zi;
        colsort[lo + pos] = i - lo;
      }
      int nrot = 0;
      const dd rho2 = dd(2.0) * rho[(size_t)l][mi];
      const int k = dc::deflate_scan<dd>(&dsort[lo], &zsort[lo], &colsort[lo], sz, rho2, &dlv[lo], &w[lo], &cnd[lo], &ddf[lo], &cdf[lo],
                                         &ra[lo], &rb[lo], &rc[lo], &rs[lo], &nrot);
      // secular roots and DELTA
      const dd rhoinv = fb::dd_recip(rho2);
      const dd* dl = &dlv[lo];
      const dd* wv = &w[lo];
      dd zz(0.0);
      for (int i = 0; i < k; ++i) zz = zz + wv[i] * wv[i];
      for (int j = 0; j < k; ++j) {
        int org = 0;
        dd tau;
        if (k == 1) {
          tau = rho2 * zz;
        } else {
          tau = dc::secular_root<dd>(dl, k, j, rho2, zz, [&](int o, dd t) {
            const dd dorg = dl[o];
            dd f(0.0);
            for (int i = 0; i < k; ++i) {
              const dd del = dc::dc_sub(dc::dc_sub(dl[i], dorg), t);
              f = f + wv[i] * (wv[i] / del);
            }
            return rhoinv + f;
          }, &org);
        }
        const dd dorg = dl[org];
        lam[lo + j] = dorg + tau;
        for (int i = 0; i < k; ++i) DEL[(size_t)(lo + j) * n + lo + i] = dc::dc_sub(dc::dc_sub(dl[i], dorg), tau);
      }
      // z-hat
      for (int i = 0; i < k; ++i) {
        dd prod = DEL[(size_t)(lo + i) * n + lo + i];
        for (int j = 0; j < k; ++j)
          if (j != i) prod = prod * (DEL[(size_t)(lo + j) * n + lo + i] / dc::dc_sub(dl[i], dl[j]));
        const dd r = sqrt(fabs(prod));
        zh[lo + i] = wv[i] < dd(0.0) ? -r : r;
      }
      // output order
      const int nd = sz - k;
      for (int t = 0; t < sz; ++t) {
        int c;
        dd val;
        if (t < k) {
          val = lam[lo + t];
          c = t;
          for (int u = 0; u < nd; ++u) c += ddf[lo + u] < val;
        } else {
          const int td = t - k;
          val = ddf[lo + td];
          c = count_less(&lam[lo], k, val, true);
          for (int u = 0; u < nd; ++u) c += (ddf[lo + u] < val) || (ddf[lo + u] == val && u < td);
        }
        outcol[lo + t] = c;
        dnew[lo + c] = val;
      }
      // vectors (the GPU sums over 128 threads in a fixed tree; here in index order)
      for (int t = 0; t < sz; ++t) {
        dd* wcol = &W[(size_t)(lo + outcol[lo + t]) * n + lo];
        if (t >= k) {
          wcol[cdf[lo + t - k]] = dd(1.0);
          continue;
        }
        const dd* dcol = &DEL[(size_t)(lo + t) * n + lo];
        dd acc(0.0);
        for (int i = 0; i < k; ++i) {
          const dd v = zh[lo + i] / dcol[i];
          acc = fb::dd_mul_add(v, v, acc);
        }
        const dd inv = fb::dd_recip(sqrt(acc));
        for (int i = 0; i < k; ++i) wcol[cnd[lo + i]] = (zh[lo + i] / dcol[i]) * inv;
      }
      // rotations
      for (int c = 0; c < sz; ++c) {
        dd* wcol = &W[(size_t)(lo + c) * n + lo];
        for (int r = nrot - 1; r >= 0; --r) {
          const int a = ra[lo + r], b = rb[lo + r];
          const dd x = wcol[a], y = wcol[b];
          wcol[a] = rc[lo + r] * x - rs[lo + r] * y;
          wcol[b] = rs[lo + r] * x + rc[lo + r] * y;
        }
      }
      // Q_new = blockdiag(Q1, Q2) W over the merge's block (the GPU's two dd GEMMs)
      for (int c = lo; c < hi; ++c)
        for (int r = lo; r < hi; ++r) {
          const int b0 = r < mid ? lo : mid, b1 = r < mid ? mid : hi;
          dd acc(0.0);
          for (int q = b0; q < b1; ++q) acc = acc + cur[(size_t)q * n + r] * W[(size_t)c * n + q];
          nxt[(size_t)c * n + r] = acc;
        }
    }
    for (int i = 0; i < n; ++i) d[i] = dnew[i];
    std::swap(cur, nxt);
  }
  for (int i = 0; i < n; ++i) {
    const dd v = d[i] * s;
    lh[i] = v.hi;
    ll[i] = v.lo;
  }
  for (size_t i = 0; i < nn; ++i) {
    qh[i] = cur[i].hi;
    ql[i] = cur[i].lo;
  }
  return 0;
}

// out[0] = max_j ||T q_j - lambda_j q_j||_2, out[1] = max |Q^T Q - I|, both accumulated in dd
extern "C" void tdd_check(const double* dh, const double* dl_, const double* eh, const double* el, int n, const double* lh,
                          const double* ll, const double* qh, const double* ql, double* out) {
  using namespace fb;
  const std::vector<dd> d = load(dh, dl_, n), e = load(eh, el, n - 1), lam = load(lh, ll, n);
  std::vector<dd> Q((size_t)n * n);
  for (size_t i = 0; i < Q.size(); ++i) Q[i] = dd(qh[i], ql[i]);
  double res = 0.0, orth = 0.0;
  for (int j = 0; j < n; ++j) {
    const dd* q = &Q[(size_t)j * n];
    dd ss(0.0);
    for (int i = 0; i < n; ++i) {
      dd r = d[i] * q[i] - lam[j] * q[i];
      if (i > 0) r = r + e[i - 1] * q[i - 1];
      if (i + 1 < n) r = r + e[i] * q[i + 1];
      ss = ss + r * r;
    }
    res = std::fmax(res, std::sqrt(ss.hi));
    for (int k = 0; k <= j; ++k) {
      dd g(0.0);
      for (int i = 0; i < n; ++i) g = g + Q[(size_t)k * n + i] * q[i];
      if (k == j) g = g - dd(1.0);
      orth = std::fmax(orth, std::fabs(g.hi + g.lo));
    }
  }
  out[0] = res;
  out[1] = orth;
}
