// Fe-statistic (Ellis, Siemens & Creighton 2012, the coherent Earth-term statistic; the reference lists it as a
// to-do: README.md:23) from the same per-(pulsar, frequency) inner products the Fp sweep forms
// (fastfp/fastfp.py:81-88): with the antenna patterns F+_p, Fx_p of a sky position the four templates of pulsar p are
//   A_p = [F+ s, F+ c, Fx s, Fx c],   s, c = sin, cos(((2 pi) f) t)          (f^(-1/3) cancels as in Fp)
//   N = sum_p [F+ N_p ; Fx N_p]                       N_p = [(s|r), (c|r)]
//   M = sum_p [[F+^2 M_p, F+ Fx M_p], [F+ Fx M_p, Fx^2 M_p]]      M_p = [[(s|s), (s|c)], [(s|c), (c|c)]]
//   Fe = 1/2 N^T M^-1 N
// so a sky scan costs one sweep (fp_sweep*_kernel with the `inner` output) plus a combine kernel: fe_combine_kernel
// writes the whole (sky position, frequency) map, fe_skymax_kernel keeps only the loudest position per frequency.
// Both form every Fe(s, f) with the two helpers below -- pulsars summed in pulsar order, general 4x4 solve with
// partial pivoting (np.linalg.solve) -- so their values agree bit for bit.
#include <cmath>

#include "../../include/fastfp_b200.h"
#include "ffp_internal.cuh"

namespace ffp {

// The arithmetic of one Fe(s, f), shared by both combine kernels. Every rounding step is written out as an intrinsic
// (__fma_rn, __dmul_rn, __ddiv_rn), so the compiler cannot contract or regroup it differently at different call sites:
// the map and the sky maximum see the same bits. They are also the bits fe_combine_kernel gave when this code was
// written with plain `a += b * c` / `a -= l * b` expressions, which the compiler fused into exactly these FMAs
// (DESIGN.md section 5c).

// Adds pulsar p's share to N and to the upper triangle of M; pp, px, xx are the rounded products fp*fp, fp*fx, fx*fx.
__device__ __forceinline__ void fe_accumulate(double (&N)[4], double (&M)[4][4], double fp, double fx, double pp,
                                              double px, double xx, double ss, double sc, double cc, double sr,
                                              double cr) {
  N[0] = __fma_rn(fp, sr, N[0]); N[1] = __fma_rn(fp, cr, N[1]);
  N[2] = __fma_rn(fx, sr, N[2]); N[3] = __fma_rn(fx, cr, N[3]);
  M[0][0] = __fma_rn(pp, ss, M[0][0]); M[0][1] = __fma_rn(pp, sc, M[0][1]); M[1][1] = __fma_rn(pp, cc, M[1][1]);
  M[0][2] = __fma_rn(px, ss, M[0][2]); M[0][3] = __fma_rn(px, sc, M[0][3]);
  M[1][2] = __fma_rn(px, sc, M[1][2]); M[1][3] = __fma_rn(px, cc, M[1][3]);
  M[2][2] = __fma_rn(xx, ss, M[2][2]); M[2][3] = __fma_rn(xx, sc, M[2][3]); M[3][3] = __fma_rn(xx, cc, M[3][3]);
}

// 0.5 N^T M^-1 N from the accumulated N and upper triangle U of M: Gaussian elimination with partial pivoting (fully
// unrolled: everything stays in registers), back substitution, then the dot product as fma(N0, x0, N1 x1) + N2 x2 + N3 x3.
__device__ __forceinline__ double fe_solve(const double (&N)[4], const double (&U)[4][4]) {
  double M[4][4] = {{U[0][0], U[0][1], U[0][2], U[0][3]}, {U[0][1], U[1][1], U[1][2], U[1][3]},
                    {U[0][2], U[1][2], U[2][2], U[2][3]}, {U[0][3], U[1][3], U[2][3], U[3][3]}};
  double b[4] = {N[0], N[1], N[2], N[3]};
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    double big = fabs(M[c][c]);
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      const double v = fabs(M[r][c]);
      if (v > big) { big = v; piv = r; }
    }
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      if (r == piv) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const double t = M[c][j]; M[c][j] = M[r][j]; M[r][j] = t; }
        const double t = b[c]; b[c] = b[r]; b[r] = t;
      }
    }
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      const double l = __ddiv_rn(M[r][c], M[c][c]);
#pragma unroll
      for (int j = c + 1; j < 4; ++j) M[r][j] = __fma_rn(-l, M[c][j], M[r][j]);
      b[r] = __fma_rn(-l, b[c], b[r]);
    }
  }
  double x[4];
#pragma unroll
  for (int r = 3; r >= 0; --r) {
    double acc = b[r];
#pragma unroll
    for (int j = r + 1; j < 4; ++j) acc = __fma_rn(-M[r][j], x[j], acc);
    x[r] = __ddiv_rn(acc, M[r][r]);
  }
  const double d = __fma_rn(N[0], x[0], __dmul_rn(N[1], x[1]));
  return __dmul_rn(0.5, __fma_rn(N[3], x[3], __fma_rn(N[2], x[2], d)));
}

__global__ void fe_combine_kernel(const double* __restrict__ inner, int P, int64_t F, const double* __restrict__ fplus,
                                  const double* __restrict__ fcross, int64_t S, double* __restrict__ out, int64_t out_ld) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t k = blockIdx.y;
  if (f >= F || k >= S) return;
  double N[4] = {0, 0, 0, 0};
  double M[4][4] = {};
  for (int p = 0; p < P; ++p) {
    const double* q = inner + ((size_t)p * F + f) * 5;
    const double ss = q[0], sc = q[1], cc = q[2], sr = q[3], cr = q[4];
    const double fp = fplus[(size_t)k * P + p], fx = fcross[(size_t)k * P + p];
    fe_accumulate(N, M, fp, fx, __dmul_rn(fp, fp), __dmul_rn(fp, fx), __dmul_rn(fx, fx), ss, sc, cc, sr, cr);
  }
  out[(size_t)k * out_ld + f] = fe_solve(N, M);
}

int launch_fe_combine(const double* d_inner, int P, int64_t F, const double* d_fplus, const double* d_fcross, int64_t S,
                      double* d_out, int64_t out_ld, cudaStream_t st) {
  if (S > 65535) { set_error("at most 65535 sky positions per call"); return FASTFP_ERR_UNSUPPORTED; }
  dim3 grid((unsigned)((F + 127) / 128), (unsigned)S);
  fe_combine_kernel<<<grid, 128, 0, st>>>(d_inner, P, F, d_fplus, d_fcross, S, d_out, out_ld);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// ---- sky maximum ------------------------------------------------------------------------------------------------
// Reduction rule, the same in every stage: a NaN loses to every other value, among equal values the lower sky index
// wins, and an all-NaN column stays (NaN, -1). It is a total order on (value, index), so the result does not depend on
// how the sky axis is split across threads, warps or CTAs.
__device__ __forceinline__ bool fe_better(double v, int64_t i, double bv, int64_t bi) {
  return !isnan(v) && (isnan(bv) || v > bv || (v == bv && i < bi));
}

// per-(sky, pulsar) weights [fp, fx, fp*fp, fp*fx, fx*fx], formed once per call
__global__ void fe_sky_weights_kernel(const double* __restrict__ fplus, const double* __restrict__ fcross, int64_t n,
                                      double* __restrict__ w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double fp = fplus[i], fx = fcross[i];
  double* o = w + i * 5;
  o[0] = fp; o[1] = fx; o[2] = __dmul_rn(fp, fp); o[3] = __dmul_rn(fp, fx); o[4] = __dmul_rn(fx, fx);
}

// A CTA owns kSkyFT frequencies (one per lane) and one contiguous chunk of the sky, which it walks in passes of
// kSkyTile positions: warp w takes positions w*kSkyKS .. w*kSkyKS+kSkyKS-1 of each pass, so a thread holds kSkyKS
// (N, M) accumulators for its frequency in registers. The pulsars go through shared memory in chunks of kSkyPC: per
// pulsar a thread reads its 5 inner products and, per sky position, the 5 weights that the whole warp reads at one
// address. Both are stored padded to 6 doubles, so each takes three 128-bit loads; at a 48-byte stride the 8 lanes of a
// 128-byte phase hit disjoint banks. When all pulsars fit in one chunk the inner products are loaded once per CTA;
// otherwise once per pass.
constexpr int kSkyFT = 32;
constexpr int kSkyWarps = 4;
constexpr int kSkyKS = 4;
constexpr int kSkyTile = kSkyWarps * kSkyKS;
constexpr int kSkyPC = 32;
constexpr int kSkyThreads = 32 * kSkyWarps;
constexpr int kSkyPad = 6;  // doubles per (pulsar, frequency) and per (pulsar, sky position) in shared memory
constexpr size_t kSkySmem = (size_t)kSkyPC * (kSkyFT + kSkyTile) * kSkyPad * sizeof(double);

__global__ void __launch_bounds__(kSkyThreads, 3)
    fe_skymax_kernel(const double* __restrict__ inner, int P, int64_t F, const double* __restrict__ w, int64_t S,
                     int64_t chunk, double* __restrict__ best_out, int64_t* __restrict__ idx_out, int64_t out_ld) {
  extern __shared__ double sh[];
  double* sh_in = sh;                                   // [kSkyPC][kSkyFT][kSkyPad]
  double* sh_w = sh + kSkyPC * kSkyFT * kSkyPad;        // [kSkyPC][kSkyTile][kSkyPad]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t f0 = (int64_t)blockIdx.x * kSkyFT;
  const int nf = F - f0 < kSkyFT ? (int)(F - f0) : kSkyFT;
  const int64_t s_begin = (int64_t)blockIdx.y * chunk;
  const int64_t s_end = min(S, s_begin + chunk);
  const bool resident = P <= kSkyPC;
  double best = kNaN();
  int64_t bidx = -1;
  for (int64_t s0 = s_begin; s0 < s_end; s0 += kSkyTile) {
    const int ns = s_end - s0 < kSkyTile ? (int)(s_end - s0) : kSkyTile;
    double N[kSkyKS][4] = {};
    double M[kSkyKS][4][4] = {};
    for (int p0 = 0; p0 < P; p0 += kSkyPC) {
      const int pc = min(kSkyPC, P - p0);
      __syncthreads();  // the previous pass is done with both buffers
      if (!resident || s0 == s_begin) {
        for (int i = threadIdx.x; i < pc * kSkyFT * 5; i += kSkyThreads) {
          const int p = i / (kSkyFT * 5), r = i - p * (kSkyFT * 5), l = r / 5;
          sh_in[(p * kSkyFT + l) * kSkyPad + (r - l * 5)] = l < nf ? inner[((size_t)(p0 + p) * F + f0) * 5 + r] : 0.0;
        }
      }
      for (int i = threadIdx.x; i < kSkyTile * pc * 5; i += kSkyThreads) {
        const int k = i / (pc * 5), r = i - k * (pc * 5), p = r / 5;
        sh_w[(p * kSkyTile + k) * kSkyPad + (r - p * 5)] = k < ns ? w[((size_t)(s0 + k) * P + p0) * 5 + r] : 0.0;
      }
      __syncthreads();
      const double2* q = reinterpret_cast<const double2*>(sh_in + lane * kSkyPad);
      const double2* wk = reinterpret_cast<const double2*>(sh_w + warp * kSkyKS * kSkyPad);
#pragma unroll 1
      for (int p = 0; p < pc; ++p, q += kSkyFT * kSkyPad / 2, wk += kSkyTile * kSkyPad / 2) {
        const double2 q0 = q[0], q1 = q[1], q2 = q[2];  // [ss, sc], [cc, sr], [cr, pad]
#pragma unroll
        for (int j = 0; j < kSkyKS; ++j) {
          const double2 a0 = wk[j * 3], a1 = wk[j * 3 + 1], a2 = wk[j * 3 + 2];  // [fp, fx], [pp, px], [xx, pad]
          fe_accumulate(N[j], M[j], a0.x, a0.y, a1.x, a1.y, a2.x, q0.x, q0.y, q1.x, q1.y, q2.x);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kSkyKS; ++j) {
      const int64_t s = s0 + warp * kSkyKS + j;
      if (s < s_end) {
        const double v = fe_solve(N[j], M[j]);
        if (fe_better(v, s, best, bidx)) { best = v; bidx = s; }
      }
    }
  }
  // merge the warps' bests of each frequency
  __syncthreads();
  double* sh_v = sh;
  int64_t* sh_i = reinterpret_cast<int64_t*>(sh + kSkyThreads);
  sh_v[threadIdx.x] = best;
  sh_i[threadIdx.x] = bidx;
  __syncthreads();
  if (warp == 0 && lane < nf) {
#pragma unroll
    for (int k = 1; k < kSkyWarps; ++k) {
      const double v = sh_v[k * 32 + lane];
      const int64_t i = sh_i[k * 32 + lane];
      if (fe_better(v, i, best, bidx)) { best = v; bidx = i; }
    }
    const size_t o = (size_t)blockIdx.y * out_ld + f0 + lane;
    best_out[o] = best;
    idx_out[o] = bidx;
  }
}

// the per-chunk bests (nchunk, F) of a split sky, merged in chunk order
__global__ void fe_skymax_merge_kernel(const double* __restrict__ part_v, const int64_t* __restrict__ part_i,
                                       int64_t nchunk, int64_t F, double* __restrict__ best_out,
                                       int64_t* __restrict__ idx_out) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  double best = part_v[f];
  int64_t bidx = part_i[f];
  for (int64_t c = 1; c < nchunk; ++c) {
    const double v = part_v[(size_t)c * F + f];
    const int64_t i = part_i[(size_t)c * F + f];
    if (fe_better(v, i, best, bidx)) { best = v; bidx = i; }
  }
  best_out[f] = best;
  idx_out[f] = bidx;
}

// ---- sky maximum of a residual batch (DESIGN.md section 5e) ---------------------------------------------------
// M(s, f) does not depend on the realisation and N_k(s, f) is linear in it: across realisations, N is the GEMM
//   [(s|r_k), (c|r_k)]  (rows (k, f), K = pulsars)  x  [F+, Fx]  (columns (s, +/x))
// on the fp64 MMA path, and M(s, f) is formed (fe_accumulate's FMAs, pulsar order) and factored (fe_solve's LU with
// partial pivoting) once per (sky, frequency) and CTA, then applied to the N_k of every realisation the CTA holds.
// A CTA owns kResRows rows (realisation, frequency) -- kt realisations x 64/kt frequencies, kt a power of two from 8
// to 64 -- and one contiguous chunk of the sky, walked in passes of kResSC positions; its (s|r), (c|r) tile crosses
// DRAM once when all pulsars fit one chunk of kResPC. Warp w holds row tiles 2(w&3), 2(w&3)+1 and column tiles
// 4(w>>2) .. +3 (4 sky positions each) of a pass. The back substitution multiplies by the reciprocal of each pivot
// instead of dividing, so values match fastfp_fe_skymax to rounding, not bit for bit.
constexpr int kResRows = 64;                 // (realisation, frequency) rows per CTA: 8 MMA row tiles
constexpr int kResSC = 32;                   // sky positions per pass: 8 MMA column tiles of 4 positions x {+, x}
constexpr int kResPC = 48;                   // pulsars per shared-memory chunk (12 k-blocks)
constexpr int kResKB = kResPC / 4;
constexpr int kResThreads = 256;
constexpr int kResWS = 2 * kResSC + 4;       // pulsar stride of the pattern tile: conflict-free B fragments
constexpr int kResFac = 17;                  // doubles per factored M: 6 multipliers, 6 of U, 4 reciprocals, pivots
constexpr size_t kResSmem = (size_t)(kResRows * kResPC * 2 + kResPC * kResWS + kResSC * 8 * kResFac) * sizeof(double);

// fe_solve's elimination on M alone: o = [l10 l20 l30 l21 l31 l32 | u01 u02 u03 u12 u13 u23 | 1/u00 .. 1/u33 | pivots]
__device__ __forceinline__ void fe_factor(const double (&U)[4][4], double* o) {
  double M[4][4] = {{U[0][0], U[0][1], U[0][2], U[0][3]}, {U[0][1], U[1][1], U[1][2], U[1][3]},
                    {U[0][2], U[1][2], U[2][2], U[2][3]}, {U[0][3], U[1][3], U[2][3], U[3][3]}};
  int code = 0, li = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int piv = c;
    double big = fabs(M[c][c]);
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      const double v = fabs(M[r][c]);
      if (v > big) { big = v; piv = r; }
    }
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      if (r == piv) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const double t = M[c][j]; M[c][j] = M[r][j]; M[r][j] = t; }
      }
    }
    code |= piv << (2 * c);
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      const double l = __ddiv_rn(M[r][c], M[c][c]);
#pragma unroll
      for (int j = c + 1; j < 4; ++j) M[r][j] = __fma_rn(-l, M[c][j], M[r][j]);
      o[li++] = l;
    }
  }
  o[6] = M[0][1]; o[7] = M[0][2]; o[8] = M[0][3]; o[9] = M[1][2]; o[10] = M[1][3]; o[11] = M[2][3];
#pragma unroll
  for (int r = 0; r < 4; ++r) o[12 + r] = __drcp_rn(M[r][r]);
  o[16] = (double)code;
}

// 0.5 N^T M^-1 N with M factored by fe_factor: fe_solve's row swaps and updates of b, then back substitution
__device__ __forceinline__ double fe_apply(const double (&N)[4], const double* o) {
  double b[4] = {N[0], N[1], N[2], N[3]};
  const int code = (int)o[16];
  int li = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int piv = (code >> (2 * c)) & 3;
#pragma unroll
    for (int r = c + 1; r < 4; ++r) {
      const bool sw = r == piv;
      const double t = sw ? b[r] : b[c];
      b[r] = sw ? b[c] : b[r];
      b[c] = t;
    }
#pragma unroll
    for (int r = c + 1; r < 4; ++r) b[r] = __fma_rn(-o[li++], b[c], b[r]);
  }
  double x[4];
  x[3] = __dmul_rn(b[3], o[15]);
  x[2] = __dmul_rn(__fma_rn(-o[11], x[3], b[2]), o[14]);
  x[1] = __dmul_rn(__fma_rn(-o[10], x[3], __fma_rn(-o[9], x[2], b[1])), o[13]);
  x[0] = __dmul_rn(__fma_rn(-o[8], x[3], __fma_rn(-o[7], x[2], __fma_rn(-o[6], x[1], b[0]))), o[12]);
  const double d = __fma_rn(N[0], x[0], __dmul_rn(N[1], x[1]));
  return __dmul_rn(0.5, __fma_rn(N[3], x[3], __fma_rn(N[2], x[2], d)));
}

__global__ void __launch_bounds__(kResThreads, 2)
    fe_skymax_res_kernel(const double* __restrict__ X, const double* __restrict__ Mi, int P, int R, int ktlog, int64_t F,
                         const double* __restrict__ fplus, const double* __restrict__ fcross, int64_t S, int64_t chunk,
                         double* __restrict__ best_out, int64_t* __restrict__ idx_out, int64_t ld, int64_t zstride) {
  extern __shared__ double sh[];
  double* sA = sh;                                   // [8 row tiles][kResKB][s|c][32]    A fragments
  double* sW = sA + kResRows * kResPC * 2;           // [kResPC][kResWS]: (F+, Fx) of each sky position of the pass
  double* sFac = sW + kResPC * kResWS;               // [64/kt frequencies][kResSC][kResFac]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wr = warp & 3, wc = warp >> 2;
  const int kt = 1 << ktlog, ft = kResRows >> ktlog;
  const int64_t f0 = (int64_t)blockIdx.x * ft;
  const int k0 = blockIdx.y * kt;
  const int64_t s_begin = (int64_t)blockIdx.z * chunk;
  const int64_t s_end = min(S, s_begin + chunk);
  const bool resident = P <= kResPC;
  const double nan = kNaN();
  // the M-stage thread of (frequency fl, sky position sl of the pass)
  const int m_fl = tid / kResSC, m_sl = tid % kResSC;
  const int64_t m_f = f0 + m_fl;
  const bool m_on = m_fl < ft && m_f < F;
  double best[2] = {nan, nan};
  int64_t bidx[2] = {-1, -1};
  for (int64_t s0 = s_begin; s0 < s_end; s0 += kResSC) {
    const int ns = s_end - s0 < kResSC ? (int)(s_end - s0) : kResSC;
    double acc[2][4][2][2] = {};
    for (int p0 = 0; p0 < P; p0 += kResPC) {
      const int pc = min(kResPC, P - p0);
      __syncthreads();  // the previous pass or chunk is done with the tiles
      if (!resident || s0 == s_begin) {
        // A fragments, walked in the order of X ([f][p][k][s|c]); rows and pulsars outside the problem are zero
        for (int i = tid; i < kResRows * kResPC * 2; i += kResThreads) {
          const int sc = i & 1, kl = (i >> 1) & (kt - 1), rest = i >> (1 + ktlog);
          const int pl = rest % kResPC, fl = rest / kResPC;
          const int row = (fl << ktlog) | kl, k = k0 + kl;
          const int64_t f = f0 + fl;
          const double v = (pl < pc && k < R && f < F) ? X[((f * P + p0 + pl) * R + k) * 2 + sc] : 0.0;
          sA[(((row >> 3) * kResKB + (pl >> 2)) * 2 + sc) * 32 + ((row & 7) << 2) + (pl & 3)] = v;
        }
      }
      for (int i = tid; i < kResSC * kResPC; i += kResThreads) {
        const int pl = i % kResPC, sl = i / kResPC;
        const bool in = pl < pc && sl < ns;
        const size_t g = (size_t)(s0 + sl) * P + p0 + pl;
        sW[pl * kResWS + 2 * sl] = in ? fplus[g] : 0.0;
        sW[pl * kResWS + 2 * sl + 1] = in ? fcross[g] : 0.0;
      }
      __syncthreads();
      if (m_on && m_sl < ns) {
        // M(s, f): fe_accumulate's M updates, pulsars in order. Between pulsar chunks the partial sums wait in this
        // thread's factor slot, so they hold no registers during the MMAs.
        double* slot = sFac + (m_fl * kResSC + m_sl) * kResFac;
        double Mu[4][4] = {};
        if (p0 > 0) {
          Mu[0][0] = slot[0]; Mu[0][1] = slot[1]; Mu[0][2] = slot[2]; Mu[0][3] = slot[3]; Mu[1][1] = slot[4];
          Mu[1][2] = slot[5]; Mu[1][3] = slot[6]; Mu[2][2] = slot[7]; Mu[2][3] = slot[8]; Mu[3][3] = slot[9];
        }
        for (int pl = 0; pl < pc; ++pl) {
          const double2 w = *reinterpret_cast<const double2*>(sW + pl * kResWS + 2 * m_sl);
          const double* q = Mi + ((size_t)m_f * P + p0 + pl) * 3;
          const double ss = __ldg(q), sc = __ldg(q + 1), cc = __ldg(q + 2);
          const double fp = w.x, fx = w.y, pp = __dmul_rn(fp, fp), px = __dmul_rn(fp, fx), xx = __dmul_rn(fx, fx);
          Mu[0][0] = __fma_rn(pp, ss, Mu[0][0]); Mu[0][1] = __fma_rn(pp, sc, Mu[0][1]);
          Mu[1][1] = __fma_rn(pp, cc, Mu[1][1]);
          Mu[0][2] = __fma_rn(px, ss, Mu[0][2]); Mu[0][3] = __fma_rn(px, sc, Mu[0][3]);
          Mu[1][2] = __fma_rn(px, sc, Mu[1][2]); Mu[1][3] = __fma_rn(px, cc, Mu[1][3]);
          Mu[2][2] = __fma_rn(xx, ss, Mu[2][2]); Mu[2][3] = __fma_rn(xx, sc, Mu[2][3]);
          Mu[3][3] = __fma_rn(xx, cc, Mu[3][3]);
        }
        if (p0 + kResPC < P) {
          slot[0] = Mu[0][0]; slot[1] = Mu[0][1]; slot[2] = Mu[0][2]; slot[3] = Mu[0][3]; slot[4] = Mu[1][1];
          slot[5] = Mu[1][2]; slot[6] = Mu[1][3]; slot[7] = Mu[2][2]; slot[8] = Mu[2][3]; slot[9] = Mu[3][3];
        } else {
          fe_factor(Mu, slot);
        }
      }
      // N: 2 row tiles x 4 column tiles x {s, c} MMAs per k-block
      const double* a_p = sA + (2 * wr) * kResKB * 64 + lane;
      const double* b_p = sW + (lane & 3) * kResWS + (4 * wc * 4 + (lane >> 3)) * 2 + ((lane >> 2) & 1);
      const int nkb = (pc + 3) >> 2;
#pragma unroll 2
      for (int kb = 0; kb < nkb; ++kb) {
        double a[2][2], b[4];
#pragma unroll
        for (int rt = 0; rt < 2; ++rt)
#pragma unroll
          for (int sc = 0; sc < 2; ++sc) a[rt][sc] = a_p[((rt * kResKB + kb) * 2 + sc) * 32];
#pragma unroll
        for (int ct = 0; ct < 4; ++ct) b[ct] = b_p[4 * kb * kResWS + ct * 8];
#pragma unroll
        for (int rt = 0; rt < 2; ++rt)
#pragma unroll
          for (int ct = 0; ct < 4; ++ct)
#pragma unroll
            for (int sc = 0; sc < 2; ++sc) dmma_m8n8k4(acc[rt][ct][sc][0], acc[rt][ct][sc][1], a[rt][sc], b[ct]);
      }
    }
    __syncthreads();  // the factors of the pass are published
#pragma unroll
    for (int rt = 0; rt < 2; ++rt) {
      const int row = 8 * (2 * wr + rt) + (lane >> 2);
      const int fl = row >> ktlog;
#pragma unroll
      for (int ct = 0; ct < 4; ++ct) {
        const int sl = 4 * (4 * wc + ct) + (lane & 3);
        if (sl >= ns) continue;
        // this lane's N: [F+ (s|r), F+ (c|r), Fx (s|r), Fx (c|r)]
        const double N[4] = {acc[rt][ct][0][0], acc[rt][ct][1][0], acc[rt][ct][0][1], acc[rt][ct][1][1]};
        const double v = fe_apply(N, sFac + (fl * kResSC + sl) * kResFac);
        if (fe_better(v, s0 + sl, best[rt], bidx[rt])) { best[rt] = v; bidx[rt] = s0 + sl; }
      }
    }
  }
  // merge the 4 lanes of a row, then the two warps of a row tile pair
#pragma unroll
  for (int rt = 0; rt < 2; ++rt)
#pragma unroll
    for (int m = 1; m <= 2; m <<= 1) {
      const double v = __shfl_xor_sync(0xffffffffu, best[rt], m);
      const int64_t i = __shfl_xor_sync(0xffffffffu, bidx[rt], m);
      if (fe_better(v, i, best[rt], bidx[rt])) { best[rt] = v; bidx[rt] = i; }
    }
  __syncthreads();
  double* sv = sh;
  int64_t* si = reinterpret_cast<int64_t*>(sh + kResRows);
  if (wc == 1 && (lane & 3) == 0)
#pragma unroll
    for (int rt = 0; rt < 2; ++rt) {
      const int row = 8 * (2 * wr + rt) + (lane >> 2);
      sv[row] = best[rt];
      si[row] = bidx[rt];
    }
  __syncthreads();
  if (wc == 0 && (lane & 3) == 0)
#pragma unroll
    for (int rt = 0; rt < 2; ++rt) {
      const int row = 8 * (2 * wr + rt) + (lane >> 2);
      if (fe_better(sv[row], si[row], best[rt], bidx[rt])) { best[rt] = sv[row]; bidx[rt] = si[row]; }
      const int k = k0 + (row & (kt - 1));
      const int64_t f = f0 + (row >> ktlog);
      if (k < R && f < F) {
        const size_t o = (size_t)blockIdx.z * zstride + (size_t)k * ld + f;
        best_out[o] = best[rt];
        idx_out[o] = bidx[rt];
      }
    }
}

static int res_ktlog(int64_t R) {
  int l = 3;
  while (l < 6 && ((int64_t)1 << l) < R) ++l;
  return l;
}

// Split of the sky axis, as fe_skymax_plan: about four rounds of the GPU at two CTAs per SM, in whole passes; one
// chunk unless may_split
FeSkyPlan fe_skymax_res_plan(int64_t F, int64_t R, int64_t S, int num_sms, bool may_split) {
  const int ktlog = res_ktlog(R);
  const int64_t ft = kResRows >> ktlog;
  const int64_t tiles = ((F + ft - 1) / ft) * ((R + (1 << ktlog) - 1) >> ktlog);
  const int64_t passes = (S + kResSC - 1) / kResSC;
  const int64_t want = may_split ? std::max<int64_t>(1, (4 * 2 * (int64_t)std::max(num_sms, 1) + tiles - 1) / tiles) : 1;
  const int64_t per = (passes + std::min(want, passes) - 1) / std::min(want, passes);
  FeSkyPlan pl;
  pl.chunk = per * kResSC;
  pl.nchunk = (passes + per - 1) / per;
  return pl;
}

int launch_fe_skymax_res(const double* d_x, const double* d_mi, int P, int64_t R, int64_t F, const double* d_fplus,
                         const double* d_fcross, int64_t S, const FeSkyPlan& pl, double* d_part_v, int64_t* d_part_i,
                         double* d_best, int64_t* d_idx, int64_t ld, cudaStream_t st) {
  FFP_CUDA(cudaFuncSetAttribute(fe_skymax_res_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kResSmem));
  const int ktlog = res_ktlog(R);
  const bool split = pl.nchunk > 1;
  dim3 grid((unsigned)((F + (kResRows >> ktlog) - 1) / (kResRows >> ktlog)), (unsigned)((R + (1 << ktlog) - 1) >> ktlog),
            (unsigned)pl.nchunk);
  fe_skymax_res_kernel<<<grid, kResThreads, kResSmem, st>>>(d_x, d_mi, P, (int)R, ktlog, F, d_fplus, d_fcross, S,
                                                            pl.chunk, split ? d_part_v : d_best, split ? d_part_i : d_idx,
                                                            split ? F : ld, split ? R * F : 0);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  if (split) {  // the per-chunk bests of every (realisation, frequency) column, merged in chunk order
    fe_skymax_merge_kernel<<<(unsigned)((R * F + 127) / 128), 128, 0, st>>>(d_part_v, d_part_i, pl.nchunk, R * F,
                                                                             d_best, d_idx);
    g_launches += 1;
    FFP_CUDA(cudaGetLastError());
  }
  return 0;
}

int launch_fe_sky_weights(const double* d_fplus,const double* d_fcross, int64_t n, double* d_w, cudaStream_t st) {
  if (n == 0) return 0;
  fe_sky_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_fplus, d_fcross, n, d_w);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// Split of the sky axis: enough CTAs for about four rounds of the GPU at three CTAs per SM, in contiguous chunks of
// whole passes. A long frequency axis alone fills the GPU and leaves the sky in one chunk.
FeSkyPlan fe_skymax_plan(int64_t F, int64_t S, int num_sms) {
  const int64_t ftiles = (F + kSkyFT - 1) / kSkyFT;
  const int64_t passes = (S + kSkyTile - 1) / kSkyTile;
  const int64_t want = std::max<int64_t>(1, (4 * 3 * (int64_t)std::max(num_sms, 1) + ftiles - 1) / ftiles);
  const int64_t per = (passes + std::min(want, passes) - 1) / std::min(want, passes);
  FeSkyPlan pl;
  pl.chunk = per * kSkyTile;
  pl.nchunk = (passes + per - 1) / per;
  return pl;
}

int launch_fe_skymax(const double* d_inner, int P, int64_t F, const double* d_w, int64_t S, const FeSkyPlan& pl,
                     double* d_part_v, int64_t* d_part_i, double* d_best, int64_t* d_idx, cudaStream_t st) {
  FFP_CUDA(cudaFuncSetAttribute(fe_skymax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSkySmem));
  const bool split = pl.nchunk > 1;
  dim3 grid((unsigned)((F + kSkyFT - 1) / kSkyFT), (unsigned)pl.nchunk);
  fe_skymax_kernel<<<grid, kSkyThreads, kSkySmem, st>>>(d_inner, P, F, d_w, S, pl.chunk, split ? d_part_v : d_best,
                                                         split ? d_part_i : d_idx, F);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  if (split) {
    fe_skymax_merge_kernel<<<(unsigned)((F + 127) / 128), 128, 0, st>>>(d_part_v, d_part_i, pl.nchunk, F, d_best,
                                                                         d_idx);
    g_launches += 1;
    FFP_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace ffp
