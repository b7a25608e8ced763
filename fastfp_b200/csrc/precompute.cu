// One-time, frequency-independent per-pulsar work for the plain-Fp path (DESIGN.md section 3):
//   Sigma = L L^T,  G = L^-1 T^T N^-1  (m x n),  u_r = G r,  w = C^-1 r = N^-1 r - G^T u_r
// and the packed, tile-contiguous layout the sweep kernel streams with one TMA bulk copy per
// chunk: packet = [ (t, 1/N, w, 0)[CI] | G in mma-fragment order (g_frag_index) ]  (CI = 16 or 32).
//
// The reference recomputes all of this for every frequency: T^T N^-1 x twice per get_xCy
// (fastfp/utils.py:51-52) and an LU solve of Sigma per call (utils.py:54), six calls per
// (frequency, pulsar) (fastfp/fastfp.py:81-88). With Sigma = L L^T,
//   (x|y) = x^T N^-1 y - (G x).(G y)        and       (x|r) = x . w
// so the per-frequency work collapses to Y = G [s c] plus five weighted dot products.
#include <algorithm>
#include <map>

#include "ffp_internal.cuh"

namespace ffp {

// In-place lower Cholesky of the m x m matrix at Lbuf + L_off (row-major; the strictly upper
// part is left untouched and never read), stopped after the first mfix columns. One CTA per
// pulsar. For a plain-Fp pack mfix = m (full factor). For an nmfp pack the leading mfix x mfix
// block becomes L_X, the lower-left block becomes Sigma_VX L_X^-T, and the trailing block is left
// holding the Schur complement TNT_VV - Sigma_VX Sigma_XX^-1 Sigma_XV (lower part).
// info[p] = j+1 if pivot j is not positive (the factor then carries NaN, which propagates like
// the reference's non-raising jnp.linalg.solve on a singular Sigma).
__global__ void chol_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                            int* __restrict__ info) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int m = pm.m;
  if (row_groups(m) > 1) return;  // wide pulsars: the blocked factorisation below
  double* A = Lbuf + pm.L_off;
  __shared__ double djj;
  for (int j = 0; j < pm.mfix; ++j) {
    if (threadIdx.x == 0) {
      const double d = A[(size_t)j * m + j];
      if (!(d > 0.0) && info[blockIdx.x] == 0) info[blockIdx.x] = j + 1;
      djj = sqrt(d);
      A[(size_t)j * m + j] = djj;
    }
    __syncthreads();
    const double d = djj;
    for (int i = j + 1 + threadIdx.x; i < m; i += blockDim.x)
      A[(size_t)i * m + j] = A[(size_t)i * m + j] / d;
    __syncthreads();
    const int cnt = m - j - 1;
    for (int idx = threadIdx.x; idx < cnt * cnt; idx += blockDim.x) {
      const int ii = idx / cnt, kk = idx - ii * cnt;
      if (kk <= ii) {
        const int i = j + 1 + ii, k = j + 1 + kk;
        A[(size_t)i * m + k] =
            fma(-A[(size_t)i * m + j], A[(size_t)k * m + j], A[(size_t)i * m + k]);
      }
    }
    __syncthreads();
  }
}

// The meta of row group k of pulsar p, a wide one (PackCore::wide, n_wide entries)
__device__ inline const PulsarMeta& group_meta(const PulsarMeta* meta, const int* wide, int n_wide, int p, int k) {
  int w = 0;
  while (wide[RG_WIDE * w] != p) ++w;
  return meta[k == 0 ? wide[RG_WIDE * w + 1] : wide[RG_WIDE * w + 2] + k - 1];
}

// ---- blocked Cholesky of the wide pulsars (row groups, DESIGN.md section 5h) -------------------------------------
// Panels of CB columns, left to right: chol_diag_kernel factors the diagonal block in shared memory, chol_panel_kernel
// solves the rows below it against that block, chol_update_kernel subtracts the panel's outer product from the
// trailing lower triangle, tile by tile over many CTAs. Every element receives exactly the operations of chol_kernel in
// the same order -- one fma per earlier column, ascending, then the division by its pivot's square root -- so the factor
// is bit for bit the unblocked one; only the work is spread over the GPU. One launch of each per panel covers every wide
// pulsar (PackCore::wide); a pulsar whose basis ends before the panel returns at once.
constexpr int CB = 32;

__global__ void chol_diag_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta, int* __restrict__ info,
                                 const int* __restrict__ wide, int k0) {
  const int p = wide[RG_WIDE * blockIdx.x];
  const PulsarMeta pm = meta[p];
  const int m = pm.m;
  if (k0 >= m) return;
  const int nb = m - k0 < CB ? m - k0 : CB;
  double* A = Lbuf + pm.L_off;
  __shared__ double s[CB][CB + 1];
  __shared__ double djj;
  for (int idx = threadIdx.x; idx < nb * nb; idx += blockDim.x) {
    const int r = idx / nb, c = idx - r * nb;
    if (c <= r) s[r][c] = A[(size_t)(k0 + r) * m + k0 + c];
  }
  __syncthreads();
  for (int j = 0; j < nb; ++j) {
    if (threadIdx.x == 0) {
      const double d = s[j][j];
      if (!(d > 0.0) && info[p] == 0) info[p] = k0 + j + 1;
      djj = sqrt(d);
      s[j][j] = djj;
    }
    __syncthreads();
    const double d = djj;
    for (int i = j + 1 + threadIdx.x; i < nb; i += blockDim.x) s[i][j] = s[i][j] / d;
    __syncthreads();
    const int cnt = nb - j - 1;
    for (int idx = threadIdx.x; idx < cnt * cnt; idx += blockDim.x) {
      const int ii = idx / cnt, kk = idx - ii * cnt;
      if (kk <= ii) s[j + 1 + ii][j + 1 + kk] = fma(-s[j + 1 + ii][j], s[j + 1 + kk][j], s[j + 1 + ii][j + 1 + kk]);
    }
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < nb * nb; idx += blockDim.x) {
    const int r = idx / nb, c = idx - r * nb;
    if (c <= r) A[(size_t)(k0 + r) * m + k0 + c] = s[r][c];
  }
}

// rows below the diagonal block: x_j = (a_j - sum_{l<j} x_l L_jl) / L_jj, one thread per row
__global__ void __launch_bounds__(64) chol_panel_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                                                        const int* __restrict__ wide, int k0) {
  const PulsarMeta pm = meta[wide[RG_WIDE * blockIdx.y]];
  const int m = pm.m;
  if (k0 + CB >= m) return;  // no rows below a full panel (a short last panel has none either)
  double* A = Lbuf + pm.L_off;
  __shared__ double l11[CB][CB + 1];
  for (int idx = threadIdx.x; idx < CB * CB; idx += blockDim.x) {
    const int r = idx / CB, c = idx - r * CB;
    l11[r][c] = c <= r ? A[(size_t)(k0 + r) * m + k0 + c] : 0.0;
  }
  __syncthreads();
  const int i = k0 + CB + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  double* Ai = A + (size_t)i * m + k0;
  double x[CB];
#pragma unroll
  for (int j = 0; j < CB; ++j) {
    double acc = Ai[j];
#pragma unroll
    for (int l = 0; l < j; ++l) acc = fma(-x[l], l11[j][l], acc);
    x[j] = acc / l11[j][j];
    Ai[j] = x[j];
  }
}

// trailing lower triangle: a_ij -= sum_l L_il L_jl over the panel's columns, ascending; 32 x 32 tiles, 2 x 2 per thread
__global__ void __launch_bounds__(256) chol_update_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                                                          const int* __restrict__ wide, int k0) {
  if (blockIdx.x > blockIdx.y) return;  // upper tiles
  const PulsarMeta pm = meta[wide[RG_WIDE * blockIdx.z]];
  const int m = pm.m, t0 = k0 + CB;
  const int i0 = t0 + 32 * blockIdx.y, j0 = t0 + 32 * blockIdx.x;
  if (i0 >= m) return;
  double* A = Lbuf + pm.L_off;
  __shared__ double Li[32][CB + 1], Lj[32][CB + 1];
  for (int idx = threadIdx.x; idx < 32 * CB; idx += blockDim.x) {
    const int r = idx / CB, c = idx - r * CB;
    Li[r][c] = i0 + r < m ? A[(size_t)(i0 + r) * m + k0 + c] : 0.0;
    Lj[r][c] = j0 + r < m ? A[(size_t)(j0 + r) * m + k0 + c] : 0.0;
  }
  __syncthreads();
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int r = ty + 16 * a, c = tx + 16 * b, i = i0 + r, j = j0 + c;
      if (i >= m || j > i) continue;
      double acc = A[(size_t)i * m + j];
#pragma unroll 8
      for (int l = 0; l < CB; ++l) acc = fma(-Li[r][l], Lj[c][l], acc);
      A[(size_t)i * m + j] = acc;
    }
}

// Where the G rows of one TOA of pulsar p (meta pm) live: in the pulsar's own packets, or, for a basis swept as row
// groups (DESIGN.md section 5h), row j of group k in the packets of that group's work item at row j - r0[k]
struct GColumn {
  double* v[MAX_RG];  // the TOA's (t, 1/N, w, 0) in each stream (null where the stream has no such TOA)
  double* g[MAX_RG];  // the G part of its packet
  int il[MAX_RG], nmb[MAX_RG], r0[MAX_RG + 1];
  int ng;
  __device__ GColumn(double* packets, const PulsarMeta* meta, const int* wide, int n_wide, const PulsarMeta& pm, int p,
                     int i) {
    ng = row_groups(pm.m);
    for (int k = 0; k < ng; ++k) {
      const PulsarMeta& it = ng == 1 ? pm : group_meta(meta, wide, n_wide, p, k);
      double* pk = packets + it.pk_off + (size_t)(i / it.ci) * (it.ci * (4 + it.mpad));
      il[k] = i % it.ci;
      v[k] = i < it.nch * it.ci ? pk + 4 * il[k] : nullptr;
      g[k] = i < it.nch * it.ci ? pk + 4 * it.ci : nullptr;
      nmb[k] = it.mpad >> 3;
      r0[k] = row_group_start(pm.m, k);
    }
    r0[ng] = pm.m;
  }
  __device__ double& at(int k, int j) const { return g[k][g_frag_index(il[k], j - r0[k], nmb[k])]; }
  // the packet stream holding row j
  __device__ int group_of(int j) const {
    int k = 0;
    while (j >= r0[k + 1]) ++k;
    return k;
  }
};

// One thread per (padded) TOA: forward-substitute L g = T_i^T / N_i and scatter t, 1/N and g into the packet layout of
// every stream that holds the pulsar's rows (GColumn); g is read back from the packets as the recurrence needs it,
// so any basis width works. Padded TOAs get zeros (weight 0: they add nothing to any sum).
__global__ void build_packets_kernel(double* __restrict__ packets,
                                     const PulsarMeta* __restrict__ meta,
                                     const double* __restrict__ Lbuf,
                                     const double* __restrict__ toas,
                                     const double* __restrict__ Nvec,
                                     const double* __restrict__ T,
                                     const int* __restrict__ slot_idx,
                                     const double* __restrict__ slot_val,
                                     const int* __restrict__ wide, int n_wide) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const GColumn gc(packets, meta, wide, n_wide, pm, blockIdx.y, i);
  const bool valid = i < pm.n;
  const double ninv = valid ? 1.0 / Nvec[pm.raw_off + i] : 0.0;
  for (int k = 0; k < gc.ng; ++k) {
    if (!gc.v[k]) continue;
    gc.v[k][0] = valid ? toas[pm.raw_off + i] : 0.0;
    gc.v[k][1] = ninv;
    gc.v[k][2] = 0.0;  // w, filled by w_kernel
    gc.v[k][3] = 0.0;
    // the stream's padding rows, and every row of a padded TOA
    for (int j = valid ? gc.r0[k + 1] - gc.r0[k] : 0; j < 8 * gc.nmb[k]; ++j)
      gc.g[k][g_frag_index(gc.il[k], j, gc.nmb[k])] = 0.0;
  }
  if (!valid) return;
  const int m = pm.m, mp = pm.mpad;
  const double* L = Lbuf + pm.L_off;
  const double* Ti = T + pm.T_off + (size_t)i * m;
  // rows below mfix: g = L_X^-1 T_X^T / N (forward substitution); rows of the per-draw block
  // (nmfp): g = T_V^T / N - (Sigma_VX L_X^-T) g_X, i.e. the same recurrence without the division
  const int mfix = pm.mfix;
  for (int kj = 0; kj < gc.ng; ++kj)
    for (int j = gc.r0[kj]; j < gc.r0[kj + 1]; ++j) {
      double acc = Ti[j] * ninv;
      const double* Lj = L + (size_t)j * m;
      const int kend = j < mfix ? j : mfix;
      for (int kk = 0; kk <= kj; ++kk) {
        const int hi = gc.r0[kk + 1] < kend ? gc.r0[kk + 1] : kend;
        for (int k = gc.r0[kk]; k < hi; ++k) acc = fma(-Lj[k], gc.at(kk, k), acc);
      }
      gc.at(kj, j) = j < mfix ? acc / Lj[j] : acc;
    }
  // block-diagonal N: the last row block holds the epoch slots; this TOA feeds sqrt(beta_e)/N_i
  // into the slot of its epoch (fp_sweep_kernel folds the slot sums when the epoch ends)
  if (slot_idx != nullptr) {
    const int sidx = slot_idx[pm.raw_off + i];
    if (sidx >= 0) gc.g[0][g_frag_index(gc.il[0], mp - 8 + sidx, gc.nmb[0])] = slot_val[pm.raw_off + i];
  }
}

// u_r[j] = sum_i G[j][i] r_i. One CTA per pulsar, one warp per basis row at a time; lanes
// stride over TOAs, fixed-order shuffle tree: deterministic.
__global__ void ur_kernel(const double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                          const double* __restrict__ res, double* __restrict__ ur, int ld, const int* __restrict__ wide,
                          int n_wide) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int j = wid; j < pm.m; j += nw) {
    // the stream holding row j: the pulsar's own packets or those of its row group
    int k = 0;
    while (j >= row_group_start(pm.m, k + 1)) ++k;
    const PulsarMeta& it = row_groups(pm.m) == 1 ? pm : group_meta(meta, wide, n_wide, blockIdx.x, k);
    const int jl = j - row_group_start(pm.m, k);
    const int CI = it.ci, mp = it.mpad, pkw = CI * (4 + mp);
    const double* pk0 = packets + it.pk_off;
    double acc = 0.0;
    for (int i = lane; i < pm.n; i += 32) {
      const double g = pk0[(size_t)(i / CI) * pkw + 4 * CI + g_frag_index(i % CI, jl, mp >> 3)];
      acc = fma(g, res[pm.raw_off + i], acc);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) ur[(size_t)blockIdx.x * ld + j] = acc;
  }
}

// w_i = r_i / N_i - sum_{j < mfix} G[j][i] u_r[j], rows in order 0 .. mfix-1 across the row groups (= (C^-1 r)_i for a
// plain-Fp pack), into the vector part of every stream that holds the pulsar's rows
__global__ void w_kernel(double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                         const double* __restrict__ res, const double* __restrict__ ur, int ld,
                         const int* __restrict__ wide, int n_wide) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pm.n) return;
  const GColumn gc(packets, meta, wide, n_wide, pm, blockIdx.y, i);
  const double* u = ur + (size_t)blockIdx.y * ld;
  double acc = 0.0;
  for (int k = 0; k < gc.ng; ++k) {
    const int hi = gc.r0[k + 1] < pm.mfix ? gc.r0[k + 1] : pm.mfix;
    for (int j = gc.r0[k]; j < hi; ++j) acc = fma(gc.at(k, j), u[j], acc);
  }
  for (int k = 0; k < gc.ng; ++k) gc.v[k][2] = res[pm.raw_off + i] * gc.v[k][1] - acc;
}

int launch_fp_precompute(fastfp_pack* pk, const double* d_toas, const double* d_res,
                         const double* d_Nvec, const double* d_T, cudaStream_t st, double* d_ur_keep,
                         const BlockNDev* bn) {
  const int P = pk->P;
  int nmax = 0, ld = MAX_M;  // ld: row length of u_r (d_ur_keep: nmfp packs, m <= MAX_M)
  for (auto& m : pk->meta) {
    nmax = m.nch * m.ci > nmax ? m.nch * m.ci : nmax;
    ld = m.m > ld ? m.m : ld;
  }
  for (auto& m : pk->items) nmax = m.nch * m.ci > nmax ? m.nch * m.ci : nmax;
  DeviceBuf<double> ur_tmp;
  double* d_ur = d_ur_keep;
  if (!d_ur) {
    FFP_CUDA(dev_alloc(&ur_tmp, (size_t)P * ld));
    d_ur = ur_tmp.get();
  }
  const PackCore& c = pk->core;
  chol_kernel<<<P, 256, 0, st>>>(c.L.get(), c.meta.get(), c.info.get());
  g_launches += 1;
  int mwide = 0;
  for (auto& m : pk->meta) mwide = row_groups(m.m) > 1 && m.m > mwide ? m.m : mwide;
  for (int k0 = 0; k0 < mwide; k0 += CB) {
    chol_diag_kernel<<<pk->n_wide, 256, 0, st>>>(c.L.get(), c.meta.get(), c.info.get(), c.wide.get(), k0);
    g_launches += 1;
    const int below = mwide - k0 - CB;
    if (below <= 0) continue;
    chol_panel_kernel<<<dim3((below + 63) / 64, pk->n_wide), 64, 0, st>>>(c.L.get(), c.meta.get(), c.wide.get(), k0);
    const int nt = (below + 31) / 32;
    chol_update_kernel<<<dim3(nt, nt, pk->n_wide), 256, 0, st>>>(c.L.get(), c.meta.get(), c.wide.get(), k0);
    g_launches += 2;
  }
  dim3 g1((nmax + 127) / 128, P);
  build_packets_kernel<<<g1, 128, 0, st>>>(c.packets.get(), c.meta.get(), c.L.get(), d_toas, d_Nvec, d_T,
                                           bn ? bn->slot_idx : nullptr, bn ? bn->slot_val : nullptr, c.wide.get(),
                                           pk->n_wide);
  ur_kernel<<<P, 256, 0, st>>>(c.packets.get(), c.meta.get(), d_res, d_ur, ld, c.wide.get(), pk->n_wide);
  // with a block-diagonal N the first term of w is N^-1 r, supplied as (N^-1 r) * Nvec
  w_kernel<<<g1, 128, 0, st>>>(c.packets.get(), c.meta.get(), bn ? bn->res_w : d_res, d_ur, ld, c.wide.get(),
                               pk->n_wide);
  g_launches += 3;
  FFP_CUDA(cudaGetLastError());
  FFP_CUDA(cudaStreamSynchronize(st));
  // the factorisation status comes back with the pack: a non-positive pivot means Sigma was not numerically
  // SPD; the factor then carries NaN, which propagates like the reference's non-raising solve -- but the
  // caller can ask which pulsar it was (fastfp_pack_factor_info; the Python mirror warns)
  pk->info.assign(P, 0);
  FFP_CUDA(cudaMemcpy(pk->info.data(), c.info.get(), sizeof(int) * P, cudaMemcpyDeviceToHost));
  return 0;
}

// ---- residual batches (DESIGN.md section 5d) ---------------------------------------------------------
// R realisations r_k of the residuals enter the sweep only through w_k = C^-1 r_k = r_k / N - G^T (G r_k). Their
// packets hold, per pulsar, the G rows of the pack and then w_1 .. w_R as rows roundup8(m) .. roundup8(m) + R - 1,
// laid out for the kernel configuration of its sweep_rows (its own CI and MP). A block-N pack has the 8 epoch-slot rows
// last, at mpad - 8, where the ECORR sweep looks for them, in the TOA layout of that configuration's chunk size
// (blockn.layout), which can differ from the pack's.

// G[j][i] of pulsar pm in the pack's packets
__device__ __forceinline__ double g_at(const double* packets, const PulsarMeta& pm, int i, int j) {
  return packets[pm.pk_off + (size_t)(i / pm.ci) * (pm.ci * (4 + pm.mpad)) + 4 * pm.ci +
                 g_frag_index(i % pm.ci, j, pm.mpad >> 3)];
}

// One thread per (padded) TOA of the residual layout: (t, 1/N, 0, 0) and the pack's G rows; all other rows zero
__global__ void res_packets_kernel(double* __restrict__ rpk, const PulsarMeta* __restrict__ rmeta,
                                   const double* __restrict__ packets, const PulsarMeta* __restrict__ meta) {
  const PulsarMeta pm = meta[blockIdx.y], rm = rmeta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int CI = rm.ci, mp = rm.mpad;
  if (i >= rm.nch * CI) return;
  double* pk = rpk + rm.pk_off + (size_t)(i / CI) * (CI * (4 + mp));
  const int il = i % CI;
  const bool valid = i < pm.n;
  const double* src = packets + pm.pk_off + (size_t)(i / pm.ci) * (pm.ci * (4 + pm.mpad)) + 4 * (i % pm.ci);
  pk[4 * il] = valid ? src[0] : 0.0;
  pk[4 * il + 1] = valid ? src[1] : 0.0;
  pk[4 * il + 2] = 0.0;  // the producers' s.w, c.w are not used in this mode
  pk[4 * il + 3] = 0.0;
  double* gp = pk + 4 * CI;
  for (int j = 0; j < mp; ++j) gp[g_frag_index(il, j, mp >> 3)] = valid && j < pm.m ? g_at(packets, pm, i, j) : 0.0;
}

// U[p][k][j] = sum_i G[j][i] r_k[i] for 8 rows x 32 realisations per CTA, TOAs staged 32 at a time. Each entry is
// summed by one thread in a fixed order (32-TOA partial sums, then their running total), so its bits do not depend
// on where its realisation sits in the batch.
__global__ void __launch_bounds__(256) ur_batch_kernel(const double* __restrict__ packets,
                                                       const PulsarMeta* __restrict__ meta,
                                                       const double* __restrict__ res, int R, int ld,
                                                       double* __restrict__ U) {
  const PulsarMeta pm = meta[blockIdx.z];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int j0 = blockIdx.x * 8, k0 = blockIdx.y * 32;
  if (j0 >= pm.m) return;
  __shared__ double Gs[8][32];
  __shared__ double Rs[32][33];
  const double* rp = res + (size_t)R * pm.raw_off;
  double acc = 0.0;
  for (int i0 = 0; i0 < pm.n; i0 += 32) {
    const int i = i0 + tx;
    Gs[ty][tx] = i < pm.n && j0 + ty < pm.m ? g_at(packets, pm, i, j0 + ty) : 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int kk = ty + 8 * q;
      Rs[kk][tx] = i < pm.n && k0 + kk < R ? rp[(size_t)(k0 + kk) * pm.n + i] : 0.0;
    }
    __syncthreads();
    double part = 0.0;
#pragma unroll 8
    for (int ii = 0; ii < 32; ++ii) part = fma(Gs[ty][ii], Rs[tx][ii], part);
    acc += part;
    __syncthreads();
  }
  if (j0 + ty < pm.m && k0 + tx < R) U[((size_t)blockIdx.z * R + k0 + tx) * ld + j0 + ty] = acc;
}

// w_k[i] = r_k[i] / N_i - sum_j G[j][i] U[k][j] (w_kernel's order) for 32 TOAs x 8 realisations per CTA, written
// straight into the residual packets: a warp takes 4 TOAs x 8 rows, i.e. one 256-byte A fragment.
__global__ void __launch_bounds__(256) w_batch_kernel(double* __restrict__ rpk, const PulsarMeta* __restrict__ rmeta,
                                                      const double* __restrict__ packets,
                                                      const PulsarMeta* __restrict__ meta,
                                                      const double* __restrict__ res, int R, int ld,
                                                      const double* __restrict__ U) {
  const PulsarMeta pm = meta[blockIdx.z], rm = rmeta[blockIdx.z];
  const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
  const int i0 = blockIdx.x * 32, k0 = blockIdx.y * 8;
  if (i0 >= pm.n) return;
  __shared__ double Gs[32][33];
  __shared__ double Us[8][33];
  const int il = 4 * wq + (lane & 3), kl = lane >> 2;
  const int i = i0 + il, k = k0 + kl;
  const double* Up = U + (size_t)blockIdx.z * R * ld;
  double acc = 0.0;
  for (int j0 = 0; j0 < pm.m; j0 += 32) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int jj = wq + 8 * q;
      Gs[jj][lane] = i0 + lane < pm.n && j0 + jj < pm.m ? g_at(packets, pm, i0 + lane, j0 + jj) : 0.0;
    }
    Us[wq][lane] = k0 + wq < R && j0 + lane < pm.m ? Up[(size_t)(k0 + wq) * ld + j0 + lane] : 0.0;
    __syncthreads();
    const int jn = pm.m - j0 < 32 ? pm.m - j0 : 32;
    for (int jj = 0; jj < jn; ++jj) acc = fma(Gs[jj][il], Us[kl][jj], acc);
    __syncthreads();
  }
  if (i >= pm.n || k >= R) return;
  const double ninv = packets[pm.pk_off + (size_t)(i / pm.ci) * (pm.ci * (4 + pm.mpad)) + 4 * (i % pm.ci) + 1];
  const double w = res[(size_t)R * pm.raw_off + (size_t)k * pm.n + i] * ninv - acc;
  const int CI = rm.ci;
  rpk[rm.pk_off + (size_t)(i / CI) * (CI * (4 + rm.mpad)) + 4 * CI +
      g_frag_index(i % CI, ((pm.m + 7) & ~7) + k, rm.mpad >> 3)] = w;
}

// Block-N residual layouts: the epoch slot of each TOA in the last row block of the residual packets (which
// res_packets_kernel left zero there), from that layout's slot indices and values
__global__ void res_slots_kernel(double* __restrict__ rpk, const PulsarMeta* __restrict__ rmeta,
                                 const int* __restrict__ slot_idx, const double* __restrict__ slot_val) {
  const PulsarMeta rm = rmeta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rm.n) return;
  const int sidx = slot_idx[rm.raw_off + i];
  if (sidx < 0) return;
  const int CI = rm.ci, mp = rm.mpad;
  rpk[rm.pk_off + (size_t)(i / CI) * (CI * (4 + mp)) + 4 * CI + g_frag_index(i % CI, mp - 8 + sidx, mp >> 3)] =
      slot_val[rm.raw_off + i];
}

bool PacketLayout::place(int p, int rows, PulsarMeta* pm) {
  KernelCfg kc{};
  if (!sweep_config(rows, &kc)) return false;
  pm->ci = kc.ci;
  pm->nch = (pm->n + kc.ci - 1) / kc.ci;
  pm->mpad = kc.mp();
  pm->pk_off = size;
  size += (int64_t)pm->nch * pm->ci * (4 + pm->mpad);
  groups[kc].push_back(p);
  return true;
}

int PacketLayout::upload(std::vector<Group>* out) const {
  for (auto& kv : groups) {
    Group g;
    g.cfg = kv.first;
    g.count = (int)kv.second.size();
    FFP_CUDA(dev_alloc(&g.pidx, (size_t)g.count));
    FFP_CUDA(cudaMemcpy(g.pidx.get(), kv.second.data(), sizeof(int) * g.count, cudaMemcpyHostToDevice));
    out->push_back(std::move(g));
  }
  return 0;
}

// the arrays of a residual batch on the device. The realisations go into (R, n_shared) blocks per pulsar at
// R * smeta.raw_off, n_shared = min(pack, residual layout) TOAs: the two layouts agree position by position on every real
// TOA (blockn.layout; with a diagonal N they are the same layout), so the pack's G rows and 1/N pair with them by
// position and the rest is padding. res_w is staged only when it is a separate array, the slot arrays only for block-N.
// A simulated batch gets the same blocks, left for sim_noise_kernel to fill.
struct ResDev {
  DeviceBuf<double> res, res_w, slot_val;
  DeviceBuf<int> slot_idx;
  DeviceBuf<PulsarMeta> smeta;  // the pack's meta with n = n_shared and raw_off into the (R, n_shared) blocks
};

static int stage_res(const ResHost& h, bool simulated, int64_t R, bool blockn, const std::vector<PulsarMeta>& smeta,
                     const std::vector<PulsarMeta>& rmeta, ResidualBatch* rb, ResDev* d, cudaStream_t st) {
  const int P = (int)smeta.size();
  const int64_t nsh = smeta.back().raw_off + smeta.back().n, nres = rmeta.back().raw_off + rmeta.back().n;
  const int64_t nchtot = rmeta.back().dm_off + rmeta.back().nch;
  const bool sep_w = simulated ? blockn : h.res_w != h.res;
  FFP_CUDA(dev_alloc(&d->res, (size_t)(R * nsh)));
  if (sep_w) FFP_CUDA(dev_alloc(&d->res_w, (size_t)(R * nsh)));
  if (blockn) {
    FFP_CUDA(dev_alloc(&d->slot_idx, (size_t)nres));
    FFP_CUDA(dev_alloc(&d->slot_val, (size_t)nres));
    FFP_CUDA(dev_alloc(&rb->done_mask, (size_t)nchtot));
  }
  FFP_CUDA(dev_alloc(&d->smeta, (size_t)P));
  FFP_CUDA(cudaMemcpyAsync(d->smeta.get(), smeta.data(), sizeof(PulsarMeta) * P, cudaMemcpyHostToDevice, st));
  for (int p = 0; p < P; ++p) {
    const PulsarMeta &sm = smeta[p], &rm = rmeta[p];
    if (!simulated)
      FFP_CUDA(cudaMemcpy2DAsync(d->res.get() + R * sm.raw_off, (size_t)sm.n * 8, h.res[p], (size_t)rm.n * 8,
                                 (size_t)sm.n * 8, (size_t)R, cudaMemcpyHostToDevice, st));
    if (sep_w && !simulated)
      FFP_CUDA(cudaMemcpy2DAsync(d->res_w.get() + R * sm.raw_off, (size_t)sm.n * 8, h.res_w[p], (size_t)rm.n * 8,
                                 (size_t)sm.n * 8, (size_t)R, cudaMemcpyHostToDevice, st));
    if (!blockn) continue;
    FFP_CUDA(cudaMemcpyAsync(d->slot_idx.get() + rm.raw_off, h.slot_idx[p], (size_t)rm.n * sizeof(int),
                             cudaMemcpyHostToDevice, st));
    FFP_CUDA(cudaMemcpyAsync(d->slot_val.get() + rm.raw_off, h.slot_val[p], (size_t)rm.n * 8, cudaMemcpyHostToDevice,
                             st));
    FFP_CUDA(cudaMemcpyAsync(rb->done_mask.get() + rm.dm_off, h.done_mask[p], (size_t)rm.nch, cudaMemcpyHostToDevice,
                             st));
  }
  return 0;
}

int build_res_packets(fastfp_pack* pk, int64_t R, const ResHost& h, cudaStream_t st, const SimHost* sim) {
  const int P = pk->P;
  const bool blockn = pk->ecorr;
  std::vector<PulsarMeta> rmeta = pk->meta, smeta = pk->meta;
  PacketLayout lay;
  int64_t raw_off = 0, sh_off = 0, dm_off = 0;
  int mmax = 0, nmax = 0, npad = 0;
  for (int p = 0; p < P; ++p) {
    PulsarMeta &rm = rmeta[p], &sm = smeta[p];
    rm.n = (int)h.n[p];
    rm.raw_off = raw_off;
    raw_off += rm.n;
    sm.n = std::min(pk->meta[p].n, rm.n);
    sm.raw_off = sh_off;
    sh_off += sm.n;
    if (!lay.place(p, sweep_rows(rm.m, R, blockn), &rm)) {
      set_error("residual batch: no kernel configuration for pulsar " + std::to_string(p));
      return FASTFP_ERR_UNSUPPORTED;
    }
    rm.dm_off = dm_off;
    dm_off += rm.nch;
    mmax = std::max(mmax, rm.m);
    nmax = std::max(nmax, sm.n);
    npad = std::max(npad, rm.nch * rm.ci);
  }
  ResidualBatch rb;
  FFP_CUDA(dev_alloc(&rb.meta, (size_t)P));
  FFP_CUDA(cudaMemcpy(rb.meta.get(), rmeta.data(), sizeof(PulsarMeta) * P, cudaMemcpyHostToDevice));
  FFP_CUDA(dev_alloc(&rb.packets, (size_t)lay.size));
  if (int rc = lay.upload(&rb.groups)) return rc;
  rb.bytes = lay.size * 8 + (int64_t)sizeof(PulsarMeta) * P + (blockn ? dm_off : 0);  // block-N: the slot masks
  ResDev d;
  if (int rc = stage_res(h, sim != nullptr, R, blockn, smeta, rmeta, &rb, &d, st)) return rc;
  SimStage ss;
  if (sim) {
    if (int rc = launch_sim_noise(*sim, pk, smeta, d.smeta.get(), R, d.res.get(), d.res_w.get(), &ss, st)) return rc;
  }
  // the first term of w_k is N^-1 r_k, supplied as (N^-1 r_k) * Nvec (as in w_kernel): r_k itself for a diagonal N
  const double* d_res_w = d.res_w ? d.res_w.get() : d.res.get();
  DeviceBuf<double> U;
  FFP_CUDA(dev_alloc(&U, (size_t)P * R * mmax));
  const PackCore& c = pk->core;
  res_packets_kernel<<<dim3((npad + 127) / 128, P), 128, 0, st>>>(rb.packets.get(), rb.meta.get(), c.packets.get(),
                                                                  d.smeta.get());
  ur_batch_kernel<<<dim3((mmax + 7) / 8, (unsigned)((R + 31) / 32), P), 256, 0, st>>>(c.packets.get(), d.smeta.get(),
                                                                                     d.res.get(), (int)R, mmax, U.get());
  // simulated: U = G n - L^-1 (sqrt(phiinv) o zeta), which turns w into C^-1 (n + T Phi^(1/2) zeta) (DESIGN.md 5g)
  if (sim && sim->noise) {
    if (int rc = launch_sim_basis(pk, R, U.get(), mmax, ss, st)) return rc;
  }
  w_batch_kernel<<<dim3((nmax + 31) / 32, (unsigned)((R + 7) / 8), P), 256, 0, st>>>(
      rb.packets.get(), rb.meta.get(), c.packets.get(), d.smeta.get(), d_res_w, (int)R, mmax, U.get());
  g_launches += 3;
  if (blockn) {
    res_slots_kernel<<<dim3((npad + 127) / 128, P), 128, 0, st>>>(rb.packets.get(), rb.meta.get(), d.slot_idx.get(),
                                                                  d.slot_val.get());
    g_launches += 1;
  }
  FFP_CUDA(cudaGetLastError());
  FFP_CUDA(cudaStreamSynchronize(st));  // U and the staging buffers are released on return
  rb.R = R;
  pk->res = std::move(rb);
  return 0;
}

}  // namespace ffp
