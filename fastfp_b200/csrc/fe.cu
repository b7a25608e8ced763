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
  double best = __longlong_as_double(0x7ff8000000000000LL);
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

int launch_fe_sky_weights(const double* d_fplus, const double* d_fcross, int64_t n, double* d_w, cudaStream_t st) {
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
