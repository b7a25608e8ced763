// fp64 pipe peak: the measured denominator for the sweep kernel's fp64 roofline
// (MEASURED_PEAKS.json carries only HBM and bf16 figures). kind 0 = DFMA, kind 1 = DMMA m16n8k4 (the shape the
// sweep kernel issues), kind 19 = DMMA m8n8k4.
#include "ffp_internal.cuh"
#include "ffp_sincos.cuh"

namespace ffp {

__global__ void __launch_bounds__(256) dfma_peak_kernel(int iters, double seed, double* sink) {
  double a[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) a[k] = seed + k + threadIdx.x * 1e-3;
  const double x = 1.0000001, y = 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 16; ++k) a[k] = fma(a[k], x, y);
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 16; ++k) s += a[k];
  if (s == 12345.678) sink[0] = s;
}

__global__ void __launch_bounds__(256) dmma_peak_kernel(int iters, double seed, double* sink) {
  double c[8][2];
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k][0] = c[k][1] = seed + k;
  const double a = 1.0 + threadIdx.x * 1e-9, b = 1e-3;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[k][0]), "+d"(c[k][1])
                   : "d"(a), "d"(b));
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1];
  if (s == 12345.678) sink[0] = s;
}

// kind 2: both instruction streams in one loop. If DMMA had its own pipe the combined rate would
// approach the sum of the two peaks; if it shares the fp64 pipe it stays at one peak.
__global__ void __launch_bounds__(256) mixed_peak_kernel(int iters, double seed, double* sink) {
  double c[4][2], a[16];
#pragma unroll
  for (int k = 0; k < 4; ++k) c[k][0] = c[k][1] = seed + k;
#pragma unroll
  for (int k = 0; k < 16; ++k) a[k] = seed + k + threadIdx.x * 1e-3;
  const double x = 1.0000001, y = 1e-9, am = 1.0 + threadIdx.x * 1e-9, bm = 1e-3;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[k][0]), "+d"(c[k][1])
                   : "d"(am), "d"(bm));
#pragma unroll
      for (int j = 0; j < 4; ++j) a[4 * k + j] = fma(a[4 * k + j], x, y);
    }
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) s += c[k][0] + c[k][1];
#pragma unroll
  for (int k = 0; k < 16; ++k) s += a[k];
  if (s == 12345.678) sink[0] = s;
}

// kind 3: register-only 9x8 outer-product accumulation (the contraction's instruction mix with no
// memory operations); kind 4: the same with the operands re-read from shared memory every step.
template <bool LDS_>
__global__ void __launch_bounds__(128, 2) outer_peak_kernel(int iters, double seed, double* sink) {
  __shared__ double sh[2][32];
  if (threadIdx.x < 64) sh[threadIdx.x >> 5][threadIdx.x & 31] = seed * 1e-3 + threadIdx.x * 1e-6;
  __syncthreads();
  double acc[9][8];
#pragma unroll
  for (int r = 0; r < 9; ++r)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[r][q] = seed + r + q;
  double a[2][9], b[2][8];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
#pragma unroll
    for (int r = 0; r < 9; ++r) a[k][r] = 1.0 + 1e-9 * (r + k + (threadIdx.x & 3));
#pragma unroll
    for (int q = 0; q < 8; ++q) b[k][q] = 1e-9 * (q + k + 1);
  }
  const int lm = (threadIdx.x >> 3) & 3, ln = threadIdx.x & 7;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (LDS_) {
        const volatile double* va = &sh[k][0];
#pragma unroll
        for (int r = 0; r < 9; ++r) a[k][r] = va[(lm + 4 * r) & 31];
#pragma unroll
        for (int q = 0; q < 8; ++q) b[k][q] = va[(ln + 8 * (q >> 1) + (q & 1)) & 31];
      }
#pragma unroll
      for (int r = 0; r < 9; ++r)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[r][q] = fma(a[k][r], b[k][q], acc[r][q]);
    }
  }
  double s = 0;
#pragma unroll
  for (int r = 0; r < 9; ++r)
#pragma unroll
    for (int q = 0; q < 8; ++q) s += acc[r][q];
  if (s == 12345.678) sink[0] = s;
}

// kind 5: one dependent DFMA chain per thread, one warp per SM sub-partition -> cycles per
// dependent fp64 op. Returned through *tflops as cycles/op (ms is the kernel time).
__global__ void __launch_bounds__(128) dfma_latency_kernel(int iters, double seed, double* sink, long long* cyc) {
  double a = seed + threadIdx.x * 1e-3;
  const double x = 1.0000001, y = 1e-9;
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 16; ++k) a = fma(a, x, y);
  }
  const long long t1 = clock64();
  if (a == 12345.678) sink[0] = a;
  if (threadIdx.x == 0 && blockIdx.x == 0) cyc[0] = t1 - t0;
}

// kinds 6-8: the producers' per-element work (phase multiply, range check, sincos_cw, the five
// weighted sums) with ILP = 1, 2, 4 independent evaluations per thread and 8 warps per SM.
// Returned through *tflops as cycles per element per warp.
template <int ILP>
__global__ void __launch_bounds__(256) sincos_rate_kernel(int iters, double seed, double* sink, long long* cyc) {
  double s2[5] = {0, 0, 0, 0, 0};
  const double omega = 6.283185307179586 * (1e-8 + threadIdx.x * 1e-11);
  double t = 4.6e9 + seed;
  const long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < ILP; ++j) {
      const double ph = __dmul_rn(omega, t + j * 86400.0);
      const bool ok = fabs(ph) <= FFP_SINCOS_MAX;
      double s, c;
      sincos_cw(ok ? ph : 0.0, &s, &c);
      const double ni = ok ? 1e13 : 0.0, wv = ok ? 1e6 : 0.0;
      const double sn = s * ni, cn = c * ni;
      s2[0] = fma(sn, s, s2[0]);
      s2[1] = fma(sn, c, s2[1]);
      s2[2] = fma(cn, c, s2[2]);
      s2[3] = fma(s, wv, s2[3]);
      s2[4] = fma(c, wv, s2[4]);
    }
    t += 1e6;
  }
  const long long t1 = clock64();
  if (s2[0] + s2[1] + s2[2] + s2[3] + s2[4] == 12345.678) sink[0] = s2[0];
  if (threadIdx.x == 0 && blockIdx.x == 0) cyc[0] = t1 - t0;
}

// kinds 9-11: the consumer's MMA pattern in isolation -- NMBW x NNB accumulator tile per warp,
// fragments re-read from shared memory for every k-block, WPS warps per SM sub-partition.
template <int NMBW, int NNB>
__global__ void __launch_bounds__(NMBW * NNB > 18 ? 128 : 512) dmma_tile_kernel(int iters, double seed, double* sink) {
  __shared__ double sh[(9 + 4) * 2 * 32];
  for (int i = threadIdx.x; i < (9 + 4) * 2 * 32; i += blockDim.x) sh[i] = seed * 1e-3 + i * 1e-9;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  double acc[NMBW][NNB][2];
#pragma unroll
  for (int r = 0; r < NMBW; ++r)
#pragma unroll
    for (int q = 0; q < NNB; ++q) acc[r][q][0] = acc[r][q][1] = seed;
  const volatile double* va = sh;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int kb = 0; kb < 2; ++kb) {
      double a[NMBW], b[NNB];
#pragma unroll
      for (int r = 0; r < NMBW; ++r) a[r] = va[(kb * 13 + r) * 32 + lane];
#pragma unroll
      for (int q = 0; q < NNB; ++q) b[q] = va[(kb * 13 + 9 + q) * 32 + lane];
#pragma unroll
      for (int r = 0; r < NMBW; ++r)
#pragma unroll
        for (int q = 0; q < NNB; ++q)
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                       : "+d"(acc[r][q][0]), "+d"(acc[r][q][1])
                       : "d"(a[r]), "d"(b[q]));
    }
  }
  double s = 0;
#pragma unroll
  for (int r = 0; r < NMBW; ++r)
#pragma unroll
    for (int q = 0; q < NNB; ++q) s += acc[r][q][0] + acc[r][q][1];
  if (s == 12345.678) sink[0] = s;
}

// kind 12: the large fp64 MMA shape m16n8k16 (sm_90+): same FMAs per 8x fewer instructions?
__global__ void __launch_bounds__(256) dmma_16816_kernel(int iters, double seed, double* sink) {
  double c[4][4];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[k][j] = seed + k + j;
  double a[8], b[4];
#pragma unroll
  for (int k = 0; k < 8; ++k) a[k] = 1.0 + (threadIdx.x + k) * 1e-9;
#pragma unroll
  for (int k = 0; k < 4; ++k) b[k] = 1e-3 * (k + 1);
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      asm volatile(
          "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
          "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
          : "+d"(c[k][0]), "+d"(c[k][1]), "+d"(c[k][2]), "+d"(c[k][3])
          : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
            "d"(b[1]), "d"(b[2]), "d"(b[3]));
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
  if (s == 12345.678) sink[0] = s;
}

// kinds 13-15: the sweep kernel's warp specialisation in isolation, registers only: 8 warps issue DMMAs
// (two per sub-partition, 8 independent accumulators each), 16 warps issue independent DFMA chains, with
// the DFMA warps asking for RATIO/256 of the pipe time the DMMA warps ask for. What the shared pipe
// delivers for such a mix is the practical ceiling of any kernel that needs both instruction kinds.
template <int RATIO256>
__global__ void __launch_bounds__(768, 1) warp_mix_kernel(int iters, double seed, double* sink) {
  const int w = threadIdx.x >> 5;
  double s = 0;
  if (w < 8) {
    double c[8][2];
#pragma unroll
    for (int k = 0; k < 8; ++k) c[k][0] = c[k][1] = seed + k;
    const double a = 1.0 + threadIdx.x * 1e-9, b = 1e-3;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(c[k][0]), "+d"(c[k][1])
                     : "d"(a), "d"(b));
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1];
  } else {
    // per iteration a DMMA warp occupies the pipe 8 x 16 = 128 cycles of its sub-partition, a DFMA warp
    // 16 x 2 = 32; two DMMA warps and four DFMA warps per sub-partition -> 256 : 128 per common iteration
    const int itf = (int)((long long)iters * 2 * RATIO256 / 256);
    double a[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) a[k] = seed + k + threadIdx.x * 1e-3;
    const double x = 1.0000001, y = 1e-9;
    for (int it = 0; it < itf; ++it) {
#pragma unroll
      for (int k = 0; k < 16; ++k) a[k] = fma(a[k], x, y);
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) s += a[k];
  }
  if (s == 12345.678) sink[0] = s;
}

// kind 16: legacy INT8 tensor MMA (mma.sync.m16n8k32.s8, int32 accumulation) from registers -- how far the
// warp-level MMA path gets on its own; the split-precision plan of DESIGN.md section 8 needs ~36 such products
// per fp64 product, so it pays only if this rate (or wgmma's) is well above 36x the fp64 pipe.
__global__ void __launch_bounds__(256) imma_peak_kernel(int iters, int seed, double* sink) {
  int c[8][4];
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k][0] = c[k][1] = c[k][2] = c[k][3] = seed + k;
  const unsigned a0 = 0x01020304u + threadIdx.x, a1 = 0x02030405u, a2 = 0x03040506u, a3 = 0x04050607u;
  const unsigned b0 = 0x01010101u, b1 = 0x02020202u;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 8; ++k)
      asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+r"(c[k][0]), "+r"(c[k][1]), "+r"(c[k][2]), "+r"(c[k][3])
                   : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
  int s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
  if (s == 123456789) sink[0] = (double)s;
}

// kinds 1, 20, 21: the 16x8 fp64 MMA shapes m16n8k{4,8,16} (sm_90+), 8 independent accumulators per warp and four
// warps per SM sub-partition, so that the MMA latency is hidden and only the issue rate of the shape remains
template <int K>
__device__ __forceinline__ void dmma_m16n8(double (&c)[4], const double (&a)[K / 2], const double (&b)[K / 4]) {
  if constexpr (K == 4)
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  else if constexpr (K == 8)
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, "
                 "{%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
                   "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <int K>
__global__ void __launch_bounds__(256, 2) dmma16_peak_kernel(int iters, double seed, double* sink) {
  double c[8][4];
#pragma unroll
  for (int k = 0; k < 8; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[k][j] = seed + k + j;
  double a[K / 2], b[K / 4];
#pragma unroll
  for (int k = 0; k < K / 2; ++k) a[k] = 1.0 + (threadIdx.x + k) * 1e-9;
#pragma unroll
  for (int k = 0; k < K / 4; ++k) b[k] = 1e-3 * (k + 1);
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int k = 0; k < 8; ++k) dmma_m16n8<K>(c[k], a, b);
  }
  double s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
  if (s == 12345.678) sink[0] = s;
}

// kinds 22, 25: kinds 13-15's warp specialisation with the sweep's m16n8k4 -- 8 warps issue m16n8k4 (8 accumulators
// each), NWD warps issue NCH independent DFMA chains each, with as many DFMAs per MMA FMA as kind 14 (the sweep kernel's
// producer ratio). Kind 22: 16 warps x 16 chains (768 threads); kind 25: 8 warps x 4 chains (512 threads, the m <= 80
// sweep's split, whose producers run four sincos chains in lockstep).
template <int NWD, int NCH>
__global__ void __launch_bounds__(32 * (8 + NWD), 1) warp_mix16_kernel(int iters, double seed, double* sink) {
  const int w = threadIdx.x >> 5;
  double s = 0;
  if (w < 8) {
    double c[8][4];
#pragma unroll
    for (int k = 0; k < 8; ++k) c[k][0] = c[k][1] = c[k][2] = c[k][3] = seed + k;
    const double a[2] = {1.0 + threadIdx.x * 1e-9, 1.0}, b[1] = {1e-3};
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int k = 0; k < 8; ++k) dmma_m16n8<4>(c[k], a, b);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s += c[k][0] + c[k][1] + c[k][2] + c[k][3];
  } else {
    // twice kind 14's DFMA iterations: a DMMA warp iteration here is 8 x 512 FMAs, there 8 x 256; the same DFMAs per
    // SM whatever NWD x NCH
    const int itf = (int)((long long)iters * 4 * 50 / 256) * (16 * 16 / (NWD * NCH));
    double a[NCH];
#pragma unroll
    for (int k = 0; k < NCH; ++k) a[k] = seed + k + threadIdx.x * 1e-3;
    const double x = 1.0000001, y = 1e-9;
    for (int it = 0; it < itf; ++it) {
#pragma unroll
      for (int k = 0; k < NCH; ++k) a[k] = fma(a[k], x, y);
    }
#pragma unroll
    for (int k = 0; k < NCH; ++k) s += a[k];
  }
  if (s == 12345.678) sink[0] = s;
}

// kinds 23, 24: the consumer's pattern with the 16x8 shapes -- NMBW basis-row blocks (B operand, one 256-byte warp
// load per k-block each) x one 16-row tile of 8 frequencies x {sin, cos} (A operand, one 128-bit load per lane and
// k-block), fragments re-read from shared memory for every k-step, two warps per SM sub-partition
template <int NMBW, int K>
__global__ void __launch_bounds__(256) dmma16_tile_kernel(int iters, double seed, double* sink) {
  constexpr int KB = K / 4;  // k-blocks of 4 per MMA
  __shared__ double sh[2 * KB * (NMBW + 2) * 32];
  for (int i = threadIdx.x; i < 2 * KB * (NMBW + 2) * 32; i += blockDim.x) sh[i] = seed * 1e-3 + i * 1e-9;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  double acc[NMBW][4];
#pragma unroll
  for (int r = 0; r < NMBW; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = seed;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const volatile double* va = sh + ks * KB * (NMBW + 2) * 32;
      double a[K / 2], b[NMBW][K / 4];
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];"
                     : "=d"(a[2 * kb]), "=d"(a[2 * kb + 1])
                     : "r"(smem_u32((const void*)(va + (kb * (NMBW + 2) + NMBW) * 32 + 2 * lane))));
#pragma unroll
        for (int r = 0; r < NMBW; ++r) b[r][kb] = va[(kb * (NMBW + 2) + r) * 32 + lane];
      }
#pragma unroll
      for (int r = 0; r < NMBW; ++r) dmma_m16n8<K>(acc[r], a, b[r]);
    }
  }
  double s = 0;
#pragma unroll
  for (int r = 0; r < NMBW; ++r) s += acc[r][0] + acc[r][1] + acc[r][2] + acc[r][3];
  if (s == 12345.678) sink[0] = s;
}

int run_fp64_peak(int kind, int iters, double* tflops, double* ms_out) {
  int dev = 0, sms = 0;
  FFP_CUDA(cudaGetDevice(&dev));
  FFP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  DeviceBuf<double> sink_buf;
  FFP_CUDA(dev_alloc(&sink_buf, 1));
  double* sink = sink_buf.get();
  Event ev0, ev1;
  FFP_CUDA(event_create(&ev0));
  FFP_CUDA(event_create(&ev1));
  cudaEvent_t e0 = ev0.get(), e1 = ev1.get();
  const int grid = sms * 8;
  float best = 1e30f;
  if (kind >= 5 && kind <= 8) {
    DeviceBuf<long long> dc_buf;
    FFP_CUDA(dev_alloc(&dc_buf, 1));
    long long* dc = dc_buf.get();
    long long hc = 0;
    for (int rep = 0; rep < 2; ++rep) {
      FFP_CUDA(cudaEventRecord(e0));
      if (kind == 5) dfma_latency_kernel<<<sms, 128>>>(iters, 1.0, sink, dc);
      else if (kind == 6) sincos_rate_kernel<1><<<sms, 256>>>(iters, 1.0, sink, dc);
      else if (kind == 7) sincos_rate_kernel<2><<<sms, 256>>>(iters, 1.0, sink, dc);
      else sincos_rate_kernel<4><<<sms, 256>>>(iters, 1.0, sink, dc);
      FFP_CUDA(cudaEventRecord(e1));
      FFP_CUDA(cudaEventSynchronize(e1));
      FFP_CUDA(cudaEventElapsedTime(&best, e0, e1));
    }
    FFP_CUDA(cudaMemcpy(&hc, dc, 8, cudaMemcpyDeviceToHost));
    g_launches += 2;
    const double per = kind == 5 ? 16.0 * iters : (kind == 6 ? 1.0 : kind == 7 ? 2.0 : 4.0) * iters;
    *tflops = (double)hc / per;
    *ms_out = best;
    return 0;
  }
  for (int rep = 0; rep < 4; ++rep) {
    FFP_CUDA(cudaEventRecord(e0));
    if (kind == 0) dfma_peak_kernel<<<grid, 256>>>(iters, 1.0, sink);
    else if (kind == 19) dmma_peak_kernel<<<grid, 256>>>(iters, 1.0, sink);
    else if (kind == 1) dmma16_peak_kernel<4><<<sms * 2, 256>>>(iters, 1.0, sink);    // 4 warps / sub-partition
    else if (kind == 20) dmma16_peak_kernel<8><<<sms * 2, 256>>>(iters, 1.0, sink);
    else if (kind == 21) dmma16_peak_kernel<16><<<sms * 2, 256>>>(iters, 1.0, sink);
    else if (kind == 22) warp_mix16_kernel<16, 16><<<sms, 768>>>(iters, 1.0, sink);
    else if (kind == 25) warp_mix16_kernel<8, 4><<<sms, 512>>>(iters, 1.0, sink);
    else if (kind == 23) dmma16_tile_kernel<9, 4><<<sms, 256>>>(iters, 1.0, sink);     // 2 warps / sub-partition
    else if (kind == 24) dmma16_tile_kernel<9, 8><<<sms, 256>>>(iters, 1.0, sink);
    else if (kind == 2) mixed_peak_kernel<<<grid, 256>>>(iters, 1.0, sink);
    else if (kind == 9) dmma_tile_kernel<9, 2><<<sms, 256>>>(iters, 1.0, sink);    // 2 warps / sub-partition
    else if (kind == 10) dmma_tile_kernel<9, 2><<<sms, 512>>>(iters, 1.0, sink);   // 4 warps / sub-partition
    else if (kind == 11) dmma_tile_kernel<9, 4><<<sms, 128>>>(iters, 1.0, sink);   // 1 warp / sub-partition
    else if (kind == 12) dmma_16816_kernel<<<sms, 256>>>(iters, 1.0, sink);
    else if (kind == 16) imma_peak_kernel<<<grid, 256>>>(iters, 1, sink);
    else if (kind == 13) warp_mix_kernel<32><<<sms, 768>>>(iters, 1.0, sink);   // DFMA asks for 1/8 of DMMA's pipe time
    else if (kind == 14) warp_mix_kernel<50><<<sms, 768>>>(iters, 1.0, sink);   // ~0.195 (the sweep kernel's mix)
    else if (kind == 15) warp_mix_kernel<96><<<sms, 768>>>(iters, 1.0, sink);   // 3/8
    else if (kind == 3) outer_peak_kernel<false><<<sms * 2, 128>>>(iters, 1.0, sink);
    else outer_peak_kernel<true><<<sms * 2, 128>>>(iters, 1.0, sink);
    FFP_CUDA(cudaEventRecord(e1));
    FFP_CUDA(cudaEventSynchronize(e1));
    float ms = 0;
    FFP_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  g_launches += 4;
  FFP_CUDA(cudaGetLastError());
  // DFMA: 16 fma/thread/iter; DMMA: 8 mma/warp/iter, 8*8*4 fma each (16*8*K for the 16x8 shapes)
  const double fma_count = kind == 0   ? (double)grid * 256 * 16.0 * iters
                           : kind == 19 ? (double)grid * 8 * 8.0 * 256.0 * iters
                           : kind == 1 || kind == 20 || kind == 21
                               ? (double)sms * 16 * 8 * (128.0 * (kind == 1 ? 4 : kind == 20 ? 8 : 16)) * iters
                           : kind == 22 || kind == 25 ? (double)sms * (8 * 8 * 512.0 * iters +
                                                         16 * 32 * 16.0 * (double)((long long)iters * 4 * 50 / 256))
                           : kind == 23 || kind == 24 ? (double)sms * 8 * 2 * 9 * (128.0 * (kind == 23 ? 4 : 8)) * iters
                           : kind == 9 ? (double)sms * 8 * 2 * 18 * 256.0 * iters
                           : kind == 10 ? (double)sms * 16 * 2 * 18 * 256.0 * iters
                           : kind == 11 ? (double)sms * 4 * 2 * 36 * 256.0 * iters
                           : kind == 12 ? (double)sms * 8 * 4 * 2048.0 * iters
                           : kind == 16 ? (double)grid * 8 * 8.0 * (16.0 * 8 * 32) * iters
                           : kind >= 13 && kind <= 15
                               ? (double)sms * (8 * 8 * 256.0 * iters +
                                                16 * 32 * 16.0 * (double)((long long)iters * 2 * (kind == 13 ? 32 : kind == 14 ? 50 : 96) / 256))
                           : kind == 2 ? (double)grid * (256 * 16.0 + 8 * 4.0 * 256.0) * iters
                                       : (double)sms * 2 * 128 * 144.0 * iters;
  *tflops = 2.0 * fma_count / (best * 1e-3) / 1e12;
  *ms_out = best;
  return 0;
}

}  // namespace ffp
