// Noise-marginalised Fp (reference fastfp/nmfp.py:57-119 under the double vmap of
// examples/run_nmfp.py:265-270) on the device.
//
// The reference rebuilds Sigma_d = TNT + diag(phiinv_d) per draw (nmfp.py:58-74) and then redoes the
// whole per-pulsar loop of calculate_Fp for every (draw, frequency). Only Sigma changes with the
// draw, and of phiinv only the trailing "varying" block (the phi layouts of nmfp.py:264-292 are
// [timing model 1e40 | fixed ECORR | red noise (+CURN)]). With the fixed columns X eliminated once
// per pulsar (Schur complement),
//     z^T Sigma_d^-1 z = |L_X^-1 z_X|^2 + z'^T S_d^-1 z',   S_d = S0 + diag(phiinv_var_d),
//     z' = z_V - Sigma_VX Sigma_XX^-1 z_X,
// so the work splits into
//   stage A (fp_sweep_kernel<NMFP=true>, once per (pulsar, frequency)): the n-long contractions --
//           the draw-independent parts a_ss, a_sc, a_cc, a_sr, a_cr and the vectors z'_s, z'_c;
//   factor  (once per (pulsar, draw)): S_d = L L^T, L^-1 in MMA-fragment order, v = L^-1 z'_r;
//   stage B (once per (pulsar, draw, frequency)): u = L^-1 z' for 32 frequencies at a time on the
//           fp64 MMA path, the five m_var-long reductions, the 2x2 solve and the pulsar sum.
#include <algorithm>
#include <cstdlib>
#include <cmath>
#include <vector>

#include "../../include/fastfp_b200.h"
#include "ffp_internal.cuh"

namespace ffp {

constexpr int NB_DT = 8;      // draws per stage-B CTA

__host__ __device__ inline int linv_blocks(int nmbv) {  // blocks (kb, mb >= kb/2) of a lower-tri L^-1
  int n = 0;
  for (int kb = 0; kb < 2 * nmbv; ++kb) n += nmbv - kb / 2;
  return n;
}
__host__ __device__ inline int linv_block_off(int nmbv, int kb) {
  int n = 0;
  for (int k = 0; k < kb; ++k) n += nmbv - k / 2;
  return n;
}

// ---- pack construction -------------------------------------------------------------------------
// L buffer <- TNT + diag(phiinv_fix) on the fixed columns (the per-draw part is added later)
__global__ void nmfp_init_sigma_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                                       const double* __restrict__ TNT, const double* __restrict__ pf) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int m = pm.m;
  for (int idx = threadIdx.x; idx < m * m; idx += blockDim.x) {
    const int i = idx / m, j = idx - i * m;
    double v = TNT[pm.L_off + idx];
    if (i == j && i < pm.mfix) v += pf[(size_t)blockIdx.x * MAX_M + i];
    Lbuf[pm.L_off + idx] = v;
  }
}

// S0[p] and z'_r[p] out of the partially factored matrix, padded to mvpad. The padding (identity rows and
// columns, zeros in z') sits at the TOP-LEFT: L^-1 of diag(I, S) is diag(I, L_S^-1), so the leading
// (mvpad - mvar) columns of L^-1 only ever multiply zeros and stage B skips their k-blocks entirely --
// with the padding at the bottom the same blocks would be spread over every block row and none could go.
__global__ void nmfp_extract_kernel(const double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                                    const double* __restrict__ ur, double* __restrict__ S0,
                                    double* __restrict__ zr, int mvpad) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int m = pm.m, mf = pm.mfix, mv = pm.mvar, pad = mvpad - mv;
  const double* A = Lbuf + pm.L_off;
  double* S = S0 + (size_t)blockIdx.x * mvpad * mvpad;
  for (int idx = threadIdx.x; idx < mvpad * mvpad; idx += blockDim.x) {
    const int i = idx / mvpad, j = idx - i * mvpad;
    double v = i == j ? 1.0 : 0.0;
    if (i >= pad && j >= pad) {
      const int ii = i - pad, jj = j - pad;
      v = ii >= jj ? A[(size_t)(mf + ii) * m + mf + jj] : A[(size_t)(mf + jj) * m + mf + ii];
    }
    S[idx] = v;
  }
  for (int k = threadIdx.x; k < mvpad; k += blockDim.x)
    zr[(size_t)blockIdx.x * mvpad + k] = k >= pad ? ur[(size_t)blockIdx.x * MAX_M + mf + k - pad] : 0.0;
}

int nmfp_pack_finish(fastfp_pack* pk, const double* d_toas, const double* d_res, const double* d_Nvec,
                     const double* d_T, const double* d_TNT, const double* d_phiinv_fix, cudaStream_t st,
                     const BlockNDev* bn) {
  const int P = pk->P;
  if (pk->mvar_max < 1) { set_error("nmfp pack: every pulsar needs at least one per-draw column (m_fix < m)"); return FASTFP_ERR_INVALID; }
  for (auto& pm : pk->meta)
    if (pm.mvar < 1) { set_error("nmfp pack: every pulsar needs at least one per-draw column (m_fix < m)"); return FASTFP_ERR_INVALID; }
  const int nmbv = pk->mvar_max <= 32 ? 4 : pk->mvar_max <= 64 ? 8 : pk->mvar_max <= 96 ? 12 : pk->mvar_max <= 128 ? 16 : 0;
  if (!nmbv) { set_error("nmfp pack: more than 128 per-draw columns (64 Fourier components) is not supported"); return FASTFP_ERR_UNSUPPORTED; }
  pk->mvpad = 8 * nmbv;
  const PackCore& c = pk->core;
  nmfp_init_sigma_kernel<<<P, 256, 0, st>>>(c.L.get(), c.meta.get(), d_TNT, d_phiinv_fix);
  g_launches += 1;
  DeviceBuf<double> d_ur;
  FFP_CUDA(dev_alloc(&d_ur, (size_t)P * MAX_M));
  int rc = launch_fp_precompute(pk, d_toas, d_res, d_Nvec, d_T, st, d_ur.get(), bn);
  if (!rc) {
    cudaError_t e = dev_alloc(&pk->nm.S0, (size_t)P * pk->mvpad * pk->mvpad);
    if (e == cudaSuccess) e = dev_alloc(&pk->nm.zr, (size_t)P * pk->mvpad);
    if (e != cudaSuccess) rc = cuda_fail(e, "nmfp pack allocation");
  }
  if (!rc) {
    nmfp_extract_kernel<<<P, 256, 0, st>>>(c.L.get(), c.meta.get(), d_ur.get(), pk->nm.S0.get(), pk->nm.zr.get(),
                                           pk->mvpad);
    g_launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = cuda_fail(e, "nmfp_extract_kernel");
    pk->bytes += (int64_t)P * pk->mvpad * (pk->mvpad + 1) * 8;
  }
  if (!rc) rc = build_i8_planes(pk, st);  // stage A on the tensor path when every pulsar fits its tile
  return rc;
}

// ---- RN_container.get_phiinv on the device ------------------------------------------------------
// phi_k = f_k^(-gamma) * (10^log10_A)^2 / 12 / pi^2 * fyr^(gamma-3) * df_k, left to right
// (nmfp.py:226-234); the CURN power law is added onto the leading entries (nmfp.py:247/275);
// phiinv = 1/phi (nmfp.py:315).
__device__ __forceinline__ double powerlaw_phi(double f, double df, double log10_A, double gamma) {
  const double fyr = 1.0 / 31557600.0;
  const double amp = pow(10.0, log10_A);
  return pow(f, -gamma) * (amp * amp) / 12.0 / 9.869604401089358 * pow(fyr, gamma - 3.0) * df;
}

__global__ void powerlaw_phiinv_kernel(const PulsarMeta* __restrict__ meta, const double* __restrict__ Ff,
                                       const double* __restrict__ dfv, const double* __restrict__ logA,
                                       const double* __restrict__ gam, int P, const double* __restrict__ cF,
                                       const double* __restrict__ cdf, int ncurn,
                                       const double* __restrict__ cA, const double* __restrict__ cG,
                                       double* __restrict__ out, int64_t ld) {
  const int d = blockIdx.x, p = blockIdx.y;
  const PulsarMeta pm = meta[p];
  const double A = logA[(size_t)d * P + p], g = gam[(size_t)d * P + p];
  for (int k = threadIdx.x; k < pm.mvar; k += blockDim.x) {
    double phi = powerlaw_phi(Ff[pm.var_off + k], dfv[pm.var_off + k], A, g);
    if (k < ncurn) phi += powerlaw_phi(cF[k], cdf[k], cA[d], cG[d]);
    out[(size_t)d * ld + pm.var_off + k] = 1.0 / phi;
  }
}

static void host_df(const double* Ff, int n, std::vector<double>& df) {
  // df = repeat(diff(concatenate(([0], Ffreqs[::2]))), 2)   (nmfp.py:226, 233)
  df.resize(n);
  double prev = 0.0;
  for (int k = 0; k < n; k += 2) {
    const double d = Ff[k] - prev;
    prev = Ff[k];
    df[k] = d;
    if (k + 1 < n) df[k + 1] = d;
  }
}

// Host side of RN_container.get_phiinv: no allocation and no synchronisation on the steady path.
// The per-draw parameters go through a pinned staging buffer owned by the pack (truly asynchronous
// copies; an event guards its reuse, so the host may run one sweep ahead of the GPU), the
// frequency tables are uploaded only when they change.
int powerlaw_phiinv_impl(const fastfp_pack* pk, const double* const* Ffreqs, const double* log10_A,
                         const double* gamma, int64_t D, const double* curn_Ffreqs, int64_t ncurn,
                         const double* curn_log10_A, const double* curn_gamma, double* out, cudaStream_t st) {
  const int P = pk->P;
  const int64_t ld = pk->mvar_total;
  const size_t nA = (size_t)D * P;
  const size_t ntab = (size_t)(2 * ld + 2 * ncurn);   // F | df | cF | cdf
  const size_t npar = 2 * nA + 2 * (size_t)D;          // A | G | cA | cG
  std::vector<double> tab(ntab), tmp;
  for (int p = 0; p < P; ++p) {
    const PulsarMeta& pm = pk->meta[p];
    if (!Ffreqs[p]) { set_error("fastfp_powerlaw_phiinv: null Ffreqs"); return FASTFP_ERR_INVALID; }
    if (ncurn > pm.mvar) { set_error("fastfp_powerlaw_phiinv: more CURN entries than per-draw columns"); return FASTFP_ERR_INVALID; }
    host_df(Ffreqs[p], pm.mvar, tmp);
    for (int k = 0; k < pm.mvar; ++k) { tab[pm.var_off + k] = Ffreqs[p][k]; tab[ld + pm.var_off + k] = tmp[k]; }
  }
  if (ncurn > 0) {
    host_df(curn_Ffreqs, (int)ncurn, tmp);
    for (int64_t k = 0; k < ncurn; ++k) { tab[2 * ld + k] = curn_Ffreqs[k]; tab[2 * ld + ncurn + k] = tmp[k]; }
  }
  PowerlawStaging& pl = pk->pl;
  if ((int64_t)(ntab + npar) > pl.cap) {
    if (pl.event) cudaEventSynchronize(pl.event.get());
    pl = {};
    FFP_CUDA(dev_alloc(&pl.dev, ntab + npar));
    FFP_CUDA(pinned_alloc(&pl.host, ntab + npar));
    FFP_CUDA(event_create(&pl.event, cudaEventDisableTiming));
    pl.cap = (int64_t)(ntab + npar);
  } else {
    FFP_CUDA(cudaEventSynchronize(pl.event.get()));  // the previous call's copies have left the staging buffer
  }
  double* dT = pl.dev.get();
  double* dP = dT + ntab;
  double* hT = pl.host.get();
  double* hP = hT + ntab;
  if (pl.tab != tab) {
    std::copy(tab.begin(), tab.end(), hT);
    FFP_CUDA(cudaMemcpyAsync(dT, hT, ntab * 8, cudaMemcpyHostToDevice, st));
    pl.tab = tab;
  }
  std::copy(log10_A, log10_A + nA, hP);
  std::copy(gamma, gamma + nA, hP + nA);
  if (ncurn > 0) {
    std::copy(curn_log10_A, curn_log10_A + D, hP + 2 * nA);
    std::copy(curn_gamma, curn_gamma + D, hP + 2 * nA + D);
  }
  FFP_CUDA(cudaMemcpyAsync(dP, hP, npar * 8, cudaMemcpyHostToDevice, st));
  FFP_CUDA(cudaEventRecord(pl.event.get(), st));
  const double *dF = dT, *dDf = dT + ld, *dcF = dT + 2 * ld, *dcdf = dcF + ncurn;
  const double *dA = dP, *dG = dP + nA, *dcA = dP + 2 * nA, *dcG = dcA + D;
  dim3 grid((unsigned)D, P);
  powerlaw_phiinv_kernel<<<grid, 64, 0, st>>>(pk->core.meta.get(), dF, dDf, dA, dG, P, dcF, dcdf, (int)ncurn, dcA, dcG,
                                               out, ld);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// ---- per-(pulsar, draw) factorisation -----------------------------------------------------------
// One warp per (pulsar, draw): S_d = S0 + diag(phiinv_var_d) = L L^T and X = L^-1 as a BLOCKED
// algorithm on the fp64 MMA path. The lower triangle lives in shared memory as 8x8 blocks (64 doubles
// each, columns XOR-swizzled so that the three access patterns below are bank-conflict free):
//   C layout   lane (R = lane/4, q = lane%4) holds [R][2q], [R][2q+1]   (mma accumulator, one 16-byte access)
//   A layout   lane holds [R][q], [R][q+4]                                (A operand; also B operand of M^T)
//   T layout   lane holds [q][R], [q+4][R]                                (B operand of M)
// Left-looking block Cholesky: block column j = (diagonal block minus the products of finished blocks)
// -> 8x8 Cholesky AND its triangular inverse in registers (warp shuffles, 8 fused steps) -> the panel
// below it times inv^T. The diagonal blocks are stored inverted (L_jj itself is never needed again).
// Then X = L^-1 block row by block row: X_ij = -inv_ii * sum_{k=j..i-1} L_ik X_kj, in place.
// X leaves in the A-fragment order stage B consumes (blocks (kb, mb >= kb/2)), v = X z'_r is formed by
// the same fragments on the way out. Only warp-level synchronisation is needed; FW warps share a CTA.
template <int NMBV>
struct FactorCfg {
  static constexpr int MV = 8 * NMBV;
  static constexpr int NBLK = NMBV * (NMBV + 1) / 2;
  static constexpr int WSZ = NBLK * 64 + MV;                       // doubles per warp: blocks + z'_r
  static constexpr int FW = NMBV <= 4 ? 8 : NMBV <= 8 ? 4 : 2;     // matrices (warps) per CTA
  static constexpr int CTAS = NMBV <= 4 ? 4 : NMBV <= 8 ? 3 : NMBV <= 12 ? 2 : 1;   // resident CTAs per SM aimed at
  static constexpr size_t SMEM = (size_t)FW * WSZ * 8;
};

// 8x8 Cholesky of the (symmetric) block held in C layout and the inverse of its factor, fused: after
// step j column j of L is final, which is all that row j of X = L^-1 needs. Returns X in C layout with
// exact zeros above the diagonal.
__device__ __forceinline__ void chol_inv_8x8(double c0, double c1, double& x0, double& x1, int lane) {
  const unsigned full = 0xffffffffu;
  const int R = lane >> 2, q = lane & 3;
  double y0 = (R == 2 * q) ? 1.0 : 0.0, y1 = (R == 2 * q + 1) ? 1.0 : 0.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const double sel = (j & 1) ? c1 : c0;  // column j lives in the lanes with q == j/2
    const int qs = j >> 1;
    const double pj = __shfl_sync(full, sel, j * 4 + qs);
    const double rinv = 1.0 / sqrt(pj);    // 1 / L[j][j]
    const double lR = __shfl_sync(full, sel, (lane & ~3) | qs) * rinv;   // L[R][j]
    const double lc0 = __shfl_sync(full, sel, (8 * q) | qs) * rinv;      // L[2q][j]
    const double lc1 = __shfl_sync(full, sel, (8 * q + 4) | qs) * rinv;  // L[2q+1][j]
    if (2 * q > j) c0 = fma(-lR, lc0, c0);
    if (2 * q + 1 > j) c1 = fma(-lR, lc1, c1);
    const double xj0 = __shfl_sync(full, y0, j * 4 + q) * rinv;  // row j of X, final
    const double xj1 = __shfl_sync(full, y1, j * 4 + q) * rinv;
    if (R > j) {
      y0 = fma(-lR, xj0, y0);
      y1 = fma(-lR, xj1, y1);
    } else if (R == j) {
      y0 = xj0;
      y1 = xj1;
    }
  }
  x0 = y0;
  x1 = y1;
}

template <int NMBV>
__global__ void __launch_bounds__(FactorCfg<NMBV>::FW * 32, FactorCfg<NMBV>::CTAS) nmfp_factor_kernel(
    const double* __restrict__ S0, const double* __restrict__ zr, const PulsarMeta* __restrict__ meta,
    const double* __restrict__ phiinv_var, int64_t ld, double* __restrict__ lf, int lfw, int P, int Db) {
  using C = FactorCfg<NMBV>;
  constexpr int MV = C::MV, FW = C::FW;
  extern __shared__ __align__(16) double sm[];
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const int64_t item = (int64_t)blockIdx.x * FW + wrp;
  if (item >= (int64_t)P * Db) return;  // whole warp leaves together
  const int d = (int)(item / P), p = (int)(item - (int64_t)d * P);
  double* W = sm + (size_t)wrp * C::WSZ;
  double* zs = W + C::NBLK * 64;
  const int R = lane >> 2, q = lane & 3;
  const int sw = (R & 2) << 1;
  const int offC = R * 8 + ((2 * q) ^ sw);           // C layout (16-byte pair)
  const int offA0 = R * 8 + (q ^ sw), offA1 = offA0 ^ 4;   // A layout
  const int offT0 = q * 8 + (R ^ ((q & 2) << 1)), offT1 = offT0 + 32;  // T layout
  auto blk = [&](int i, int j) { return W + (i * (i + 1) / 2 + j) * 64; };
  auto ld_c = [&](const double* b, double& v0, double& v1) {
    const double2 t = *reinterpret_cast<const double2*>(b + offC);
    v0 = t.x; v1 = t.y;
  };
  auto st_c = [&](double* b, double v0, double v1) { *reinterpret_cast<double2*>(b + offC) = make_double2(v0, v1); };

  const PulsarMeta pm = meta[p];
  const double* S = S0 + (size_t)p * MV * MV;
  const double* ph = phiinv_var + (size_t)d * ld + pm.var_off;
#pragma unroll
  for (int i = 0; i < NMBV; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      double2 t = __ldg(reinterpret_cast<const double2*>(S + (size_t)(8 * i + R) * MV + 8 * j + 2 * q));
      if (i == j && 8 * i + R >= MV - pm.mvar) {  // real rows follow the top padding
        const double pv = ph[8 * i + R - (MV - pm.mvar)];
        if (R == 2 * q) t.x += pv;
        if (R == 2 * q + 1) t.y += pv;
      }
      st_c(blk(i, j), t.x, t.y);
    }
  }
  for (int i = lane; i < MV; i += 32) zs[i] = zr[(size_t)p * MV + i];
  __syncwarp();

  // ---- block Cholesky (left-looking), diagonal blocks stored inverted ----
#pragma unroll
  for (int j = 0; j < NMBV; ++j) {
    double bj[NMBV > 1 ? NMBV - 1 : 1][2];  // A layout of the finished blocks of row j
#pragma unroll
    for (int k = 0; k < j; ++k) { bj[k][0] = blk(j, k)[offA0]; bj[k][1] = blk(j, k)[offA1]; }
    double c0, c1, t0 = 0.0, t1 = 0.0;
    ld_c(blk(j, j), c0, c1);
#pragma unroll
    for (int k = 0; k < j; ++k) { dmma_m8n8k4(t0, t1, bj[k][0], bj[k][0]); dmma_m8n8k4(t0, t1, bj[k][1], bj[k][1]); }
    double x0, x1;
    chol_inv_8x8(c0 - t0, c1 - t1, x0, x1, lane);
    st_c(blk(j, j), x0, x1);
    // panel, part 1: A_ij - sum_k L_ik L_jk^T
#pragma unroll
    for (int i = j + 1; i < NMBV; ++i) {
      double u0 = 0.0, u1 = 0.0, v0, v1;
#pragma unroll
      for (int k = 0; k < j; ++k) {
        dmma_m8n8k4(u0, u1, blk(i, k)[offA0], bj[k][0]);
        dmma_m8n8k4(u0, u1, blk(i, k)[offA1], bj[k][1]);
      }
      ld_c(blk(i, j), v0, v1);
      st_c(blk(i, j), v0 - u0, v1 - u1);
    }
    __syncwarp();
    // panel, part 2: times inv_jj^T (B operand of M^T = A layout of M)
    if (j + 1 < NMBV) {
      const double bi0 = blk(j, j)[offA0], bi1 = blk(j, j)[offA1];
      double pa[NMBV > 1 ? NMBV - 1 : 1][2];
#pragma unroll
      for (int i = j + 1; i < NMBV; ++i) { pa[i - j - 1][0] = blk(i, j)[offA0]; pa[i - j - 1][1] = blk(i, j)[offA1]; }
      __syncwarp();
#pragma unroll
      for (int i = j + 1; i < NMBV; ++i) {
        double r0 = 0.0, r1 = 0.0;
        dmma_m8n8k4(r0, r1, pa[i - j - 1][0], bi0);
        dmma_m8n8k4(r0, r1, pa[i - j - 1][1], bi1);
        st_c(blk(i, j), r0, r1);
      }
      __syncwarp();
    }
  }

  // ---- X = L^-1, block row by block row, in place ----
#pragma unroll
  for (int i = 1; i < NMBV; ++i) {
    double la[NMBV > 1 ? NMBV - 1 : 1][2];
#pragma unroll
    for (int k = 0; k < i; ++k) { la[k][0] = blk(i, k)[offA0]; la[k][1] = blk(i, k)[offA1]; }
    const double nx0 = -blk(i, i)[offA0], nx1 = -blk(i, i)[offA1];
    __syncwarp();
#pragma unroll
    for (int j = 0; j < i; ++j) {
      double t0 = 0.0, t1 = 0.0;
#pragma unroll
      for (int k = j; k < i; ++k) {
        dmma_m8n8k4(t0, t1, la[k][0], blk(k, j)[offT0]);
        dmma_m8n8k4(t0, t1, la[k][1], blk(k, j)[offT1]);
      }
      st_c(blk(i, j), t0, t1);
    }
    __syncwarp();
    double tb[NMBV > 1 ? NMBV - 1 : 1][2];
#pragma unroll
    for (int j = 0; j < i; ++j) { tb[j][0] = blk(i, j)[offT0]; tb[j][1] = blk(i, j)[offT1]; }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < i; ++j) {
      double r0 = 0.0, r1 = 0.0;
      dmma_m8n8k4(r0, r1, nx0, tb[j][0]);
      dmma_m8n8k4(r0, r1, nx1, tb[j][1]);
      st_c(blk(i, j), r0, r1);
    }
    __syncwarp();
  }

  // ---- out: A-fragment blocks (kb, mb >= kb/2) and v = X z'_r from the same fragments ----
  double* out = lf + ((size_t)d * P + p) * lfw;
  double acc[NMBV][2];
#pragma unroll
  for (int mb = 0; mb < NMBV; ++mb) acc[mb][0] = acc[mb][1] = 0.0;
  int b = 0;
#pragma unroll
  for (int kb = 0; kb < 2 * NMBV; ++kb) {
    const double zb = zs[4 * kb + q];
#pragma unroll
    for (int mb = kb / 2; mb < NMBV; ++mb, ++b) {
      const double val = blk(mb, kb / 2)[(kb & 1) ? offA1 : offA0];
      out[b * 32 + lane] = val;
      dmma_m8n8k4(acc[mb][0], acc[mb][1], val, zb);
    }
  }
  if (q == 0) {
#pragma unroll
    for (int mb = 0; mb < NMBV; ++mb) out[b * 32 + 8 * mb + R] = acc[mb][0];
  }
}

// ---- stage B ------------------------------------------------------------------------------------
struct StageBArgs {
  const double* Z;       // [P][nt32][MV*64]   z' tiles (B-fragment order)
  const double* A;       // [P][nt32][160]     a_ss | a_sc | a_cc | a_sr | a_cr, 32 frequencies each
  const double* lf;      // [Db][P][lfw]       L^-1 fragments + v
  const double* freqs;   // [F]
  const PulsarMeta* meta;  // per pulsar: mvar -> leading padding k-blocks that are skipped
  double* out;           // [D][F]  (this launch writes rows d0 .. d0+Db-1)
  int64_t F, out_ld;
  int P, nt32, Db, lfw;
  int nt_blk;            // Z and A hold blocks of nt_blk tiles: [block][P][nt_blk] (one block = nt32 when they were made here;
                         // one block per rank when the tiles were made frequency-sharded and all-gathered)
};

// One CTA = NH half-tiles of 32 frequencies x NB_DT draws, all pulsars. 8*NH consumer warps (4
// frequencies each: one n8 MMA column block holds their sin and cos columns) plus one producer warp
// whose lane 0 drives the TMA rings: the z' tile of a pulsar (double-buffered, reused by the NB_DT draws)
// and the L^-1 fragments of each (pulsar, draw) (NS stages). Full/empty mbarriers only -- no CTA-wide
// barrier in the loop, so the warps drift apart by up to NS iterations and the epilogue of one warp
// (shuffles, the batched 2x2 solves) overlaps the MMAs of the others.
template <int NMBV>
struct StageBCfg {
  static constexpr int MV = 8 * NMBV, ZT = MV * 64;
  static constexpr int NH = NMBV <= 8 ? 2 : 1;                 // 32-frequency half-tiles per CTA
  static constexpr int NS = NMBV <= 8 ? 4 : NMBV <= 12 ? 3 : 2;  // L^-1 ring depth
  static constexpr int ZBUF = NMBV <= 12 ? 2 : 1;              // z' tile buffers (128 columns: one 64 KB tile fits)
  static constexpr int NWB = 8 * NH;                           // consumer warps
  static constexpr int THREADS = 32 * (NWB + 1);
  static constexpr int LFW = (NMBV * (NMBV + 1)) * 32 + MV;    // linv_blocks(NMBV) * 32 + MV
  static constexpr size_t SMEM = (size_t)(ZBUF * NH * ZT + ZBUF * NH * 160 + NS * LFW) * 8 + (size_t)(4 + 2 * NS) * 8;
  static_assert(SMEM <= 227 * 1024, "stage B shared memory");
};

template <int NMBV>
__global__ void __launch_bounds__(StageBCfg<NMBV>::THREADS, 1) nmfp_stageB_kernel(const StageBArgs ar) {
  using C = StageBCfg<NMBV>;
  constexpr int KBV = 2 * NMBV, ZT = C::ZT, NH = C::NH, NS = C::NS, NWB = C::NWB, LFW = C::LFW, ZBUF = C::ZBUF;
  extern __shared__ __align__(128) unsigned char raw[];
  double* Zb = reinterpret_cast<double*>(raw);       // [ZBUF][NH][ZT]
  double* Ab = Zb + ZBUF * NH * ZT;                  // [ZBUF][NH][160]
  double* Lb = Ab + ZBUF * NH * 160;                 // [NS][LFW]
  uint64_t* zfull = reinterpret_cast<uint64_t*>(Lb + NS * LFW);  // [2]
  uint64_t* zempty = zfull + 2;                                  // [2]
  uint64_t* lfull = zempty + 2;                                  // [NS]
  uint64_t* lempty = lfull + NS;                                 // [NS]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int t32 = blockIdx.x * NH;                   // first 32-frequency tile of this CTA
  const int nh = min(NH, ar.nt32 - t32);             // half-tiles that exist (the last CTA may hold one)
  const int d0 = blockIdx.y * NB_DT;
  const int nd = min(NB_DT, ar.Db - d0);
  const int nit = ar.P * nd;
  if (tid == 0) {
    for (int s = 0; s < 2; ++s) { mbar_init(&zfull[s], 1); mbar_init(&zempty[s], NWB); }
    for (int s = 0; s < NS; ++s) { mbar_init(&lfull[s], 1); mbar_init(&lempty[s], NWB); }
    fence_barrier_init();
  }
  __syncthreads();

  if (w == NWB) {  // ---- producer ----
    if (lane != 0) return;
    for (int it = 0; it < nit; ++it) {
      const int p = it / nd, dl = it - p * nd;
      if (dl == 0) {  // z' tile(s) and the a-terms of pulsar p, before the first L^-1 of that pulsar
        const int buf = p % ZBUF;
        if (p >= ZBUF) mbar_wait(&zempty[buf], ((p / ZBUF) - 1) & 1);
        mbar_expect_tx(&zfull[buf], (uint32_t)(nh * (ZT + 160) * 8));
        const size_t tile = ((size_t)(t32 / ar.nt_blk) * ar.P + p) * ar.nt_blk + (size_t)(t32 % ar.nt_blk);
        tma_load_1d(Zb + buf * NH * ZT, ar.Z + tile * ZT, (uint32_t)(nh * ZT * 8), &zfull[buf]);
        tma_load_1d(Ab + buf * NH * 160, ar.A + tile * 160, (uint32_t)(nh * 160 * 8), &zfull[buf]);
      }
      const int s = it % NS;
      if (it >= NS) mbar_wait(&lempty[s], ((it / NS) - 1) & 1);
      mbar_expect_tx(&lfull[s], LFW * 8);
      tma_load_1d(Lb + s * LFW, ar.lf + ((size_t)(d0 + dl) * ar.P + p) * ar.lfw, LFW * 8, &lfull[s]);
    }
    return;
  }

  // ---- consumers ----
  const int h = w >> 3, wl = w & 7;                  // half-tile, warp inside it
  // B fragment of lane (k = lane & 3, n = lane >> 2) in one (k-block, column block) of a z' tile, the layout
  // NmfpTiles::z writes: row k, sin (n even) or cos (n odd) of frequency n / 2 of the column block
  const int bperm = 16 * ((lane >> 2) & 1) + 4 * (lane >> 3) + (lane & 3);
  constexpr int nblk = NMBV * (NMBV + 1);
  const int fi = 4 * wl + (lane & 3);                // this lane group's frequency inside the half-tile
  const int64_t f = (int64_t)(t32 + h) * 32 + fi;
  const double fval = f < ar.F ? ar.freqs[f] : 1.0;
  // The 2x2 solves are batched: after the xor-reduction every lane holds the five sums of its frequency
  // (lane & 3); the lanes with (lane >> 2) == dl keep those of draw dl, and once the NB_DT draws of a
  // pulsar are through, all 32 lanes solve at once (one (frequency, draw) each) instead of 4 lanes per
  // iteration -- the fp64 pipe is charged per warp instruction, not per active lane.
  static_assert(NB_DT == 8, "lane >> 2 indexes the draw inside a CTA");
  double fpacc = 0.0;
  double k0 = 0.0, k1 = 0.0, k2 = 0.0, k3 = 0.0, k4 = 0.0;
  int kb0 = 0;

  for (int it = 0; it < nit; ++it) {
    const int p = it / nd, dl = it - p * nd, buf = p % ZBUF, s = it % NS;
    if (dl == 0) mbar_wait_spin(&zfull[buf], (p / ZBUF) & 1);
    mbar_wait_spin(&lfull[s], (it / NS) & 1);
    const double* zt = Zb + (buf * NH + h) * ZT + wl * 32 + bperm;
    const double* lt = Lb + s * LFW;
    if (dl == 0) kb0 = (8 * NMBV - ar.meta[p].mvar) >> 2;  // k-blocks that only see the top padding
    double acc[NMBV][2];
#pragma unroll
    for (int mb = 0; mb < NMBV; ++mb) acc[mb][0] = acc[mb][1] = 0.0;
#pragma unroll
    for (int kb = 0; kb < KBV; ++kb) {
      if (kb >= kb0) {  // warp-uniform
        const double b = zt[kb * 8 * 32];
        const int off = linv_block_off(NMBV, kb);
#pragma unroll
        for (int mb = kb / 2; mb < NMBV; ++mb)
          dmma_m8n8k4(acc[mb][0], acc[mb][1], lt[(off + mb - kb / 2) * 32 + lane], b);
      }
    }
    // u = L^-1 z' for row 8*mb + (lane>>2), frequency fi: [0] = sin, [1] = cos
    const double* v = lt + nblk * 32;
    double r5[5] = {0, 0, 0, 0, 0};
#pragma unroll
    for (int mb = 0; mb < NMBV; ++mb) {
      const double us = acc[mb][0], uc = acc[mb][1], vv = v[8 * mb + (lane >> 2)];
      r5[0] = fma(us, us, r5[0]);
      r5[1] = fma(us, uc, r5[1]);
      r5[2] = fma(uc, uc, r5[2]);
      r5[3] = fma(us, vv, r5[3]);
      r5[4] = fma(uc, vv, r5[4]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&lempty[s]);  // this warp is done with the L^-1 stage
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      r5[k] += __shfl_xor_sync(0xffffffffu, r5[k], 4);
      r5[k] += __shfl_xor_sync(0xffffffffu, r5[k], 8);
      r5[k] += __shfl_xor_sync(0xffffffffu, r5[k], 16);
    }
    if ((lane >> 2) == dl) { k0 = r5[0]; k1 = r5[1]; k2 = r5[2]; k3 = r5[3]; k4 = r5[4]; }
    if (dl == nd - 1) {  // uniform: the draws of pulsar p are complete
      const double* a = Ab + (buf * NH + h) * 160 + fi;
      const double m00 = a[0] - k0, m01 = a[32] - k1, m11 = a[64] - k2;
      const double N0 = a[96] - k3, N1 = a[128] - k4;
      __syncwarp();
      if (lane == 0) mbar_arrive(&zempty[buf]);  // z' tile and a-terms of pulsar p are consumed
      fpacc += term_2x2(m00, m01, m11, N0, N1);  // pulsar sum in pulsar order, starting from 0 (nmfp.py:98,117)
    }
  }
  if ((lane >> 2) < nd && f < ar.F) {
    double val = fpacc;
    if (!(fval > 0.0)) val = kNaN();
    ar.out[(size_t)(d0 + (lane >> 2)) * ar.out_ld + f] = val;
  }
}

// Events between the stages of one sweep (only when the caller asked for stage timing): the interval
// ending at a mark is charged to that mark's stage (0 = stage A incl. clears, 1 = factor, 2 = stage B).
struct StageMarks {
  bool on = false;
  std::vector<std::pair<Event, int>> ev;
  void mark(int stage, cudaStream_t st) {
    if (!on) return;
    Event e;
    if (event_create(&e) != cudaSuccess) return;
    cudaEventRecord(e.get(), st);
    ev.emplace_back(std::move(e), stage);
  }
  void finish(cudaStream_t st, double* ms3) {
    if (!on) return;
    cudaStreamSynchronize(st);
    ms3[0] = ms3[1] = ms3[2] = 0.0;
    for (size_t i = 1; i < ev.size(); ++i) {
      float t = 0.f;
      if (ev[i].second >= 0 && cudaEventElapsedTime(&t, ev[i - 1].first.get(), ev[i].first.get()) == cudaSuccess)
        ms3[ev[i].second] += t;
    }
    ev.clear();
  }
};

template <int NMBV>
static int run_factor_and_stageB(const fastfp_pack* pk, const double* d_phiinv, int64_t ld, int Db,
                                 StageBArgs sb, double* d_lf, cudaStream_t st, StageMarks& marks) {
  const size_t fsm = FactorCfg<NMBV>::SMEM;
  static bool attr_done[64] = {};
  const size_t bsm = StageBCfg<NMBV>::SMEM;
  if (sb.lfw != StageBCfg<NMBV>::LFW) { set_error("internal: L^-1 fragment width mismatch"); return FASTFP_ERR_UNSUPPORTED; }
  if (!attr_done[pk->device & 63]) {
    FFP_CUDA(cudaFuncSetAttribute(nmfp_factor_kernel<NMBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsm));
    FFP_CUDA(cudaFuncSetAttribute(nmfp_stageB_kernel<NMBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsm));
    attr_done[pk->device & 63] = true;
  }
  constexpr int FW = FactorCfg<NMBV>::FW;
  const unsigned gf = (unsigned)(((int64_t)pk->P * Db + FW - 1) / FW);
  nmfp_factor_kernel<NMBV><<<gf, FW * 32, fsm, st>>>(pk->nm.S0.get(), pk->nm.zr.get(), pk->core.meta.get(), d_phiinv,
                                                   ld, d_lf, sb.lfw, pk->P, Db);
  marks.mark(1, st);
  dim3 gb((sb.nt32 + StageBCfg<NMBV>::NH - 1) / StageBCfg<NMBV>::NH, (Db + NB_DT - 1) / NB_DT);
  nmfp_stageB_kernel<NMBV><<<gb, StageBCfg<NMBV>::THREADS, bsm, st>>>(sb);
  marks.mark(2, st);
  g_launches += 2;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// Stage A alone: the z' tiles and a-terms of F frequencies into Z [P][ceil(F/32)][MV*64] and A [P][ceil(F/32)][160].
int nmfp_stage_a_impl(const fastfp_pack* pk, const double* d_freqs, int64_t F, double* dZ, double* dA, cudaStream_t st) {
  const int P = pk->P, MV = pk->mvpad;
  const int nt32 = (int)((F + 31) / 32);
  // stage-A tiles are written sparsely (rows of narrower pulsars, the tail of the last tile): clear
  FFP_CUDA(cudaMemsetAsync(dZ, 0, (size_t)P * nt32 * (MV * 64) * 8, st));
  FFP_CUDA(cudaMemsetAsync(dA, 0, (size_t)P * nt32 * 160 * 8, st));
  // on the tensor path when the pack carries digit planes, else on the fp64 DMMA kernel
  return launch_sweep(pk, d_freqs, F, NmfpTiles{dZ, dA, MV}, st);
}

// Factor + stage B for D draws on tiles that already exist: Z and A hold blocks of nt_blk tiles ([block][P][nt_blk]),
// together the ceil(F/32) tiles of the F frequencies. out: (D, F) rows with leading dimension out_ld.
int nmfp_stage_b_impl(const fastfp_pack* pk, const double* d_freqs, int64_t F, const double* dZ, const double* dA,
                      int nt_blk, const double* d_phiinv_var, int64_t D, double* d_out, int64_t out_ld, cudaStream_t st,
                      StageMarks& marks) {
  const int P = pk->P, MV = pk->mvpad, NMBV = MV / 8;
  const int lfw = linv_blocks(NMBV) * 32 + MV;
  const int nt32 = (int)((F + 31) / 32);
  if (nt_blk <= 0 || (nt_blk < nt32 && (nt_blk & 1))) {  // a CTA reads two consecutive tiles: never across blocks
    set_error("stage B: tiles per block must be even when the tiles come in several blocks");
    return FASTFP_ERR_INVALID;
  }
  // Draw batches bound the L^-1 store (written by the factor kernel, read by every frequency tile of stage B). One batch
  // of up to 1.5 GiB is the fastest (C3: 17.7 ms, 2.4 GB of DRAM traffic per sweep, far from binding at ~130 GB/s);
  // FASTFP_B200_NMFP_LF_MB=64 keeps the store L2-resident instead (batches of whole CTA waves: 0.79 GB per sweep, the
  // rest being the z' tiles re-read per batch, at 18.1 ms) -- bytes, not time, so it is not the default.
  static const long lf_mb = getenv("FASTFP_B200_NMFP_LF_MB") ? atol(getenv("FASTFP_B200_NMFP_LF_MB")) : 0;
  const int64_t per_draw = (int64_t)P * lfw * 8;
  int64_t DB;
  if (lf_mb <= 0) {
    DB = std::max<int64_t>(NB_DT, std::min<int64_t>(D, ((3LL << 26) / ((int64_t)P * lfw)) / NB_DT * NB_DT));
  } else {
    int64_t groups = std::max<int64_t>(1, (lf_mb << 20) / (per_draw * NB_DT));          // draw groups that fit the budget
    const int64_t pairs = (nt32 + 1) / 2;                                                 // CTAs per draw group (NMBV <= 8)
    if (pairs < pk->num_sms) {                                                            // round down to whole waves
      const int64_t per_wave = std::max<int64_t>(1, pk->num_sms / pairs);
      if (groups >= per_wave) groups = groups / per_wave * per_wave;
    }
    DB = std::min<int64_t>(std::max<int64_t>(NB_DT, groups * NB_DT), std::max<int64_t>(NB_DT, (D + NB_DT - 1) / NB_DT * NB_DT));
  }
  if (int rc = pk->lf.grow(DB * P * lfw)) return rc;
  double* dLf = pk->lf.get();
  for (int64_t dd = 0; dd < D; dd += DB) {
    const int Db = (int)std::min(DB, D - dd);
    StageBArgs sb{dZ, dA, dLf, d_freqs, pk->core.meta.get(), d_out + dd * out_ld, F, out_ld, P, nt32, Db, lfw,
                  nt_blk};
    const double* ph = d_phiinv_var + dd * pk->mvar_total;
    int rc;
    if (NMBV == 4) rc = run_factor_and_stageB<4>(pk, ph, pk->mvar_total, Db, sb, dLf, st, marks);
    else if (NMBV == 8) rc = run_factor_and_stageB<8>(pk, ph, pk->mvar_total, Db, sb, dLf, st, marks);
    else if (NMBV == 12) rc = run_factor_and_stageB<12>(pk, ph, pk->mvar_total, Db, sb, dLf, st, marks);
    else rc = run_factor_and_stageB<16>(pk, ph, pk->mvar_total, Db, sb, dLf, st, marks);
    if (rc) return rc;
  }
  return 0;
}

int nmfp_stage_b_only(const fastfp_pack* pk, const double* d_freqs, int64_t F, const double* dZ, const double* dA,
                      int nt_blk, const double* d_phiinv_var, int64_t D, double* d_out, cudaStream_t st) {
  StageMarks marks;  // (stage timing is a facility of the combined sweep)
  return nmfp_stage_b_impl(pk, d_freqs, F, dZ, dA, nt_blk, d_phiinv_var, D, d_out, F, st, marks);
}

int nmfp_sweep_impl(const fastfp_pack* pk, const double* d_freqs, int64_t F, const double* d_phiinv_var,
                    int64_t D, double* d_out, cudaStream_t st) {
  const int P = pk->P, MV = pk->mvpad;
  // frequency batches bound the stage-A outputs (1 GiB)
  const int64_t per_f32 = (int64_t)P * (MV * 64 + 160);
  int64_t FB = std::max<int64_t>(32, ((1LL << 27) / std::max<int64_t>(1, per_f32)) * 32);
  FB = std::min<int64_t>(FB, (F + 31) / 32 * 32);
  const int64_t nt32_max = FB / 32;
  if (int rc = pk->scratch.grow(P * nt32_max * (int64_t)(MV * 64 + 160))) return rc;
  double* dZ = pk->scratch.get();
  double* dA = dZ + P * nt32_max * (int64_t)MV * 64;
  StageMarks marks;
  marks.on = pk->time_stages;
  marks.mark(-1, st);
  for (int64_t f0 = 0; f0 < F; f0 += FB) {
    const int64_t Fb = std::min(FB, F - f0);
    if (int rc = nmfp_stage_a_impl(pk, d_freqs + f0, Fb, dZ, dA, st)) return rc;
    marks.mark(0, st);
    if (int rc = nmfp_stage_b_impl(pk, d_freqs + f0, Fb, dZ, dA, (int)((Fb + 31) / 32), d_phiinv_var, D, d_out + f0, F, st,
                                   marks)) return rc;
  }
  marks.finish(st, pk->stage_ms);
  return 0;
}

}  // namespace ffp
