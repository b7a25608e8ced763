// The frequency-sweep kernel on the INT8 tensor cores: Y = G [s c] as an error-free product of 8-bit digit planes
// (Hopper wgmma.mma_async .s32.s8.s8, exact int32 accumulation in registers), everything else in fp64.
//
// Replaces the body of FastFp.calculate_Fp under jax.vmap (reference fastfp/fastfp.py:69-92, examples/run_fp.py:63)
// like fp_sweep_kernel.cuh does, for packs with n <= 16384 TOAs per pulsar, a diagonal N and up to 639 basis columns
// (128 operand rows -- 127 columns + the C^-1 r row -- per pass over the TOAs; wider bases take one pass per row group
// of 128, the b-sums adding up in the epilogue); the fp64 DMMA kernel stays as the path for everything else. fp64 has
// no wgmma kind, and the DMMA formulation shares the fp64 pipe with the sincos generation (DESIGN.md section 4.6); the
// INT8 tensor path is a different unit altogether, and integer accumulation is exact.
//
// Number format (radix 256, 7 planes per operand, validated at the level of the statistic by
// tests/test_split_precision_emulation.py):
//   G row j (and the extra row w = C^-1 r):  g = G / 2^e_j with |g| < 1/4,  Qg = rint(g 2^55),
//        Qg = sum_i d_i 256^(6-i), balanced digits d_i in [-128, 127]  (pack time, i8_planes_kernel)
//   s, c in [-1, 1]:  Q = rint(x 2^54) = sum_j v_j 256^(6-j), balanced digits (producers: an exponent add and one
//        F2I.S64.F64; the bytes of Q + 0x80..80 are the digits + 128)
//   Y_j = 2^(e_j - 13) sum_{g=0..6} 256^-g  sum_{i+j=g} sum_k d_i(k) v_j(k):   28 plane products, one int32
//        accumulator per weight g (|d v| <= 2^14, 7 products per TOA: exact for n <= 18 724 TOAs)
//
// One 640-thread CTA per SM, static round-robin over (pulsar, 16-frequency tile) work items, per stage of 32 TOAs:
//   warpgroup 0, warp 0 lane 0: TMA -- one bulk copy of the stage's G planes (7 x rows x 32 bytes, already in the
//            SWIZZLE_32B K-major operand layout) and one of its (t, 1/N) vectors, mbarrier rings
//   warpgroups 1-2 (consumers, operand rows 0-63 and 64-127 of the row group): 28 wgmma m64n32k32 (N = 32: 16
//            frequencies x {sin, cos}, K = 32 TOAs) into the 7 register accumulators (7 x 16 registers per thread);
//            after the last stage of a pass the same warpgroup runs the epilogue: fp64 recombination,
//            b = Y_s.Y_s, Y_s.Y_c, Y_c.Y_c over the basis rows, (s|r), (c|r) from the w row, pivoted 2x2 solve
//            (jnp.linalg.solve at fastfp.py:90)
//   warpgroups 3-4 (producers, one per stage, alternating): sincos_cw of ((2 pi) f) t (fastfp.py:78-79 phase order),
//            the digit split, 14 conflict-free 4-byte stores per thread into the B-operand planes, and the fp64
//            sums s N^-1 s, s N^-1 c (c N^-1 c = sum 1/N - s N^-1 s)
// The accumulators of a 128 x 32 tile fill 112 registers of each of the 256 consumer threads, which is what sets the
// tile at 16 frequencies: 32 would need the whole register file.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../include/fastfp_b200.h"
#include "ffp_internal.cuh"
#include "ffp_sincos.cuh"

namespace ffp {
namespace i8 {

constexpr int NPL = 7;                 // digit planes per operand
constexpr int KT = 32;                 // TOAs per stage = K bytes per operand row (one SWIZZLE_32B atom wide)
constexpr int NF = 16;                 // frequencies per work item
constexpr int NBR = 2 * NF;            // rows of the B operand: row = 16 * {0: sin, 1: cos} + frequency
constexpr int S_PLANE = NBR * KT;      // 1024 bytes
constexpr int S_STAGE = NPL * S_PLANE; // 7168 bytes
constexpr int V_STAGE = KT * 16;       // (t, 1/N) per TOA
constexpr int SST = 8, VST = 8;        // ring depths (even: a slot is always served by the same producer group)
constexpr int RS = 640;                // row-scale stride per pulsar: up to 5 row groups of 128 operand rows (m <= 639)
constexpr int NCONS = 2;               // consumer warpgroups (64 operand rows each)
constexpr int NACC = 16;               // accumulator registers per thread per weight: 64 x 32 / 128
// Warp layout: warpgroup 0 control (TMA), 1-2 consumers, 3-4 producers (one group of 4 warps per stage, thread = one
// frequency x four TOAs, the two groups alternating stages). setmaxnreg moves registers between the warpgroups.
constexpr int THREADS = 640;
constexpr int NPW = 8;                 // producer warps
constexpr int REGS_LAUNCH = 96;        // 65536 / THREADS, multiple of 8
constexpr int REGS_CTRL = 32, REGS_CONS = 152, REGS_PROD = 72;
static_assert(128 * REGS_CTRL + 256 * REGS_CONS + 32 * NPW * REGS_PROD <= THREADS * REGS_LAUNCH, "register pool");
static_assert(SST % 2 == 0 && VST % 2 == 0, "ring depths must be even");

struct Args {
  const unsigned char* planes;   // per pulsar, per stage: [V_STAGE bytes (t, 1/N)] then per row group [NPL][rows_g][32] swizzled
  const double* rowscale;        // [P][RS]  2^(e_j - 13), 0 for rows that do not exist
  const PulsarMeta* meta;
  const int* pidx;
  const double* freqs;
  int64_t F;
  FpOut fp;                      // fp_sweep_i8_kernel<false>
  NmfpTiles nm;                  // fp_sweep_i8_kernel<true>: nmfp stage A
  int ntile, nwork;              // 16-frequency tiles per pulsar, work items
  int nt32;                      // 32-frequency tiles of the nmfp outputs
  int gslot, gst;                // G ring: bytes per slot (7 x rows_max x 32), number of slots
};

// byte offset of (row r, K byte c) in a K-major tile with 32-byte rows, SWIZZLE_32B: 8-row groups of 256 bytes, the
// 16-byte chunk index XORed with bit 2 of the row (validated by tools/probes/umma_i8_split_check.cu)
__host__ __device__ inline int swz32(int r, int c) {
  return (r >> 3) * 256 + (r & 7) * 32 + ((((c >> 4) ^ ((r & 7) >> 2)) & 1) << 4) + (c & 15);
}

// ---- pack time: digit planes of G (+ the w row) --------------------------------------------------------------
// e_j from the row maximum: |G_j / 2^e_j| < 1/4; rs_j = 2^(e_j - 13). bad[p] is set when a row holds a non-finite
// value (singular Sigma, NaN data): the integer planes could not carry it, so such a pack stays on the fp64 path.
__global__ void i8_rowscale_kernel(const double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                                   double* __restrict__ rowscale, int* __restrict__ rowexp, int* __restrict__ bad) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int r = blockIdx.x;
  if (r >= RS || pm.i8_nst == 0) return;  // (pulsars the tensor sweep does not take have no stages)
  double* rs = rowscale + (size_t)blockIdx.y * RS + r;
  int* re = rowexp + (size_t)blockIdx.y * RS + r;
  if (r > pm.m) {
    if (threadIdx.x == 0) { *rs = 0.0; *re = 0; }
    return;
  }
  const int CI = pm.ci, mp = pm.mpad, pkw = CI * (4 + mp);
  const double* pk0 = packets + pm.pk_off;
  double mx = 0.0;
  bool nonfinite = false;
  for (int i = threadIdx.x; i < pm.n; i += blockDim.x) {
    const double* pk = pk0 + (size_t)(i / CI) * pkw;
    const int il = i % CI;
    const double v = r < pm.m ? pk[4 * CI + g_frag_index(il, r, mp >> 3)] : pk[4 * il + 2];  // G row or w
    const double a = fabs(v);
    if (!(a <= 1.7e308)) nonfinite = true;
    mx = fmax(mx, a);
  }
  __shared__ double smx[32];
  __shared__ int snf;
  if (threadIdx.x == 0) snf = 0;
  __syncthreads();
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) smx[threadIdx.x >> 5] = mx;
  if (nonfinite) atomicOr(&snf, 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, smx[w]);
    int e = 0;
    if (mx > 0.0) {
      int x;
      frexp(mx, &x);  // mx = f 2^x, f in [1/2, 1)  ->  |G| < 2^x
      e = x + 2;
    }
    *re = e;
    *rs = mx > 0.0 ? scalbn(1.0, e - 13) : 0.0;
    if (snf) atomicOr(&bad[blockIdx.y], 1);
  }
}

// one CTA per (stage, pulsar): the (t, 1/N) vectors and the 7 x rows x 32 digit bytes of the stage
__global__ void i8_planes_kernel(const double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                                 const int* __restrict__ rowexp, unsigned char* __restrict__ planes) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int st = blockIdx.x;
  if (st >= pm.i8_nst) return;
  const int rows = pm.i8_rows, CI = pm.ci, mp = pm.mpad, pkw = CI * (4 + mp);
  const double* pk0 = packets + pm.pk_off;
  unsigned char* out = planes + pm.i8_off + (size_t)st * (V_STAGE + NPL * rows * KT);
  double2* v = reinterpret_cast<double2*>(out);
  for (int kk = threadIdx.x; kk < KT; kk += blockDim.x) {
    const int i = st * KT + kk;
    double2 tv = make_double2(0.0, 0.0);  // padded TOAs: weight 0 (and zero digits below)
    if (i < pm.n) {
      const double* pk = pk0 + (size_t)(i / CI) * pkw;
      tv = make_double2(pk[4 * (i % CI)], pk[4 * (i % CI) + 1]);
    }
    v[kk] = tv;
  }
  // row groups of 128 operand rows (one accumulator set each, one pass over the TOAs per group): group-major, then
  // plane-major, so that a (stage, group) is one contiguous TMA copy
  unsigned char* g = out + V_STAGE;
  const int* re = rowexp + (size_t)blockIdx.y * RS;
  for (int e = threadIdx.x; e < rows * KT; e += blockDim.x) {
    const int r = e / KT, kk = e - r * KT;
    const int i = st * KT + kk;
    double val = 0.0;
    if (i < pm.n && r <= pm.m) {
      const double* pk = pk0 + (size_t)(i / CI) * pkw;
      const int il = i % CI;
      val = r < pm.m ? pk[4 * CI + g_frag_index(il, r, mp >> 3)] : pk[4 * il + 2];
    }
    // Qg = rint(val 2^(55 - e)): exact scaling, |Qg| <= 2^53; balanced base-256 digits = bytes of Qg + 0x80..80, - 128
    const long long Q = __double2ll_rn(scalbn(val, 55 - re[r]));
    const unsigned long long U = (unsigned long long)(Q + 0x0080808080808080LL) ^ 0x0080808080808080ULL;
    const int grp = r >> 7, rl = r & 127, rows_g = min(128, rows - 128 * grp);
    unsigned char* gg = g + (size_t)grp * (NPL * 128 * KT);
    const int off = swz32(rl, kk);
#pragma unroll
    for (int p = 0; p < NPL; ++p) gg[(size_t)p * rows_g * KT + off] = (unsigned char)(U >> (8 * (6 - p)));
  }
}


// ---- device helpers ------------------------------------------------------------------------------------------
// wgmma shared-memory descriptor: K-major, SWIZZLE_32B (layout type 3), stride between 8-row groups 256 bytes; the
// leading-byte offset is unused for swizzled K-major operands one atom wide. Operand bases are 1024-byte aligned.
constexpr uint64_t DESC_HI = ((uint64_t)(256 >> 4) << 32) | ((uint64_t)3 << 62);
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr >> 4) & 0x3fffu) | (1u << 16); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// D (64 x 32, s32) = A (64 x 32 s8, K-major) B^T (32 x 32 s8, K-major) + (accumulate ? D : 0)
__device__ __forceinline__ void wgmma_i8(uint32_t (&d)[NACC], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(da), "l"(db), "r"(accumulate));
}

// x in [-1, 1] -> the 7 bytes of Q + 0x80..80, Q = rint(x 2^54), every byte XORed with 0x80: balanced signed digits,
// most significant in byte 6. The scaling is an integer add on the exponent field (zero and subnormals land below
// 2^-900 and round to 0; the fast path is entered for finite data only) and the rounding ONE conversion instruction
// (F2I.S64.F64), which keeps the producers off the fp64 pipe for this part; an all-integer extraction costs ~30
// instructions per value.
__device__ __forceinline__ uint2 digits7(double x) {
  const long long Q = __double2ll_rn(__hiloint2double(__double2hiint(x) + (54 << 20), __double2loint(x)));
  const long long U = Q + 0x0080808080808080LL;
  return make_uint2((uint32_t)U ^ 0x80808080u, (uint32_t)((unsigned long long)U >> 32) ^ 0x00808080u);
}

// Every wait of this kernel is bounded (wait_wd below): a protocol error would otherwise hang the GPU; a timed-out wait
// reports where it was stuck and traps, which the host sees as a launch failure instead of a hung device.
__device__ __forceinline__ void wait_timeout(int tag, uint32_t k) {
  printf("[fastfp_b200 i8 sweep] mbarrier wait timed out: tag %d, stage/item %u, block %d, warp %d\n", tag, k,
         (int)blockIdx.x, (int)(threadIdx.x >> 5));
  __trap();
}
// mbarrier.try_wait with a suspend-time hint: the warp sleeps in hardware until the phase completes or HINT_NS pass
// (without the hint the time slice is a few tens of nanoseconds, so waiting warps would spend issue slots polling).
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t* bar, uint32_t parity, uint32_t hint_ns) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
      " selp.b32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));  // volatile: stays inside the branch that asks for it
  return t;
}
// SLEEP_NS = 0: the waiter is on the critical path and polls with the default time slice; otherwise each poll may
// suspend the warp for up to SLEEP_NS, so that waiting warps do not spend issue slots the producers need. Bounded: no
// legitimate wait is longer than one item (< 1 ms); after 5 s on the global timer (looked at every 256 polls) the CTA
// reports where it was stuck and traps.
template <int SLEEP_NS>
__device__ __forceinline__ void wait_wd(uint64_t* bar, uint32_t parity, int tag, uint32_t k) {
  if (mbar_try_wait(bar, parity)) return;
  uint32_t n = 0;
  unsigned long long t0 = 0;
  while (!(SLEEP_NS ? mbar_try_wait_hint(bar, parity, (uint32_t)SLEEP_NS) : mbar_try_wait(bar, parity))) {
    if ((++n & 255u) == 0) {
      const unsigned long long t = global_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > 5000000000ULL) wait_timeout(tag, k);
    }
  }
}

// The 28 products of one 32-TOA stage for one consumer warpgroup: accumulator g = i + j collects plane i of G times
// plane j of [s c]; the first product into accumulator g of a pass is (0, g). Descriptors differ in their address
// field only, so each is one add on the low word of the stage's base descriptor.
__device__ __forceinline__ void issue_stage(uint32_t (&acc)[NPL][NACC], uint32_t da_lo, uint32_t db_lo,
                                            uint32_t aplane16, bool first_stage) {
#pragma unroll
  for (int i = 0; i < NPL; ++i) {
#pragma unroll
    for (int j = 0; j < NPL - i; ++j)
      wgmma_i8(acc[i + j], DESC_HI | (uint64_t)(da_lo + (uint32_t)i * aplane16),
               DESC_HI | (uint64_t)(db_lo + (uint32_t)j * (S_PLANE >> 4)), (!first_stage || i > 0) ? 1u : 0u);
  }
}

struct Smem {
  unsigned char *G, *S, *V;
  double *redA;          // [2][2][NF][3] producer sums: buffer, producer group, frequency
  double *part;          // [8][NF][3]    epilogue partial b-sums per consumer warp
  double *nval;          // [NF][2]       (s|r), (c|r) from the w row
  uint64_t *g_full, *g_empty, *v_full, *v_empty, *s_full, *s_empty, *sums_full, *sums_empty;
  __device__ Smem(unsigned char* raw, const Args& ar) {
    G = raw;
    S = G + (size_t)ar.gst * ar.gslot;
    V = S + SST * S_STAGE;
    redA = reinterpret_cast<double*>(V + VST * V_STAGE);
    part = redA + 2 * 2 * NF * 3;
    nval = part + 8 * NF * 3;
    g_full = reinterpret_cast<uint64_t*>(nval + NF * 2);
    g_empty = g_full + 8;
    v_full = g_empty + 8;
    v_empty = v_full + VST;
    s_full = v_empty + VST;
    s_empty = s_full + SST;
    sums_full = s_empty + SST;
    sums_empty = sums_full + 2;
  }
};
constexpr size_t SMEM_FIXED = (size_t)SST * S_STAGE + VST * V_STAGE + (2 * 2 * NF * 3 + 8 * NF * 3 + NF * 2) * 8 +
                              (8 + 8 + 2 * VST + 2 * SST + 4) * 8;

template <bool NMFP>
__global__ void __launch_bounds__(THREADS, 1) fp_sweep_i8_kernel(const Args ar) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  Smem sm(smem_raw, ar);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < ar.gst; ++s) { mbar_init(&sm.g_full[s], 1); mbar_init(&sm.g_empty[s], NCONS); }
    for (int s = 0; s < VST; ++s) { mbar_init(&sm.v_full[s], 1); mbar_init(&sm.v_empty[s], 4); }
    for (int s = 0; s < SST; ++s) { mbar_init(&sm.s_full[s], 4); mbar_init(&sm.s_empty[s], NCONS); }
    for (int b = 0; b < 2; ++b) { mbar_init(&sm.sums_full[b], NPW); mbar_init(&sm.sums_empty[b], 1); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wid < 4) {
    // ================= control warpgroup: TMA (warp 0, lane 0) =================
    reg_dealloc<REGS_CTRL>();
    if (wid == 0 && lane == 0) {
      // ring positions and phase parities are carried incrementally (no division by the runtime ring depth per stage)
      uint32_t k = 0, sv = 0, vpar = 0, sg = 0, gpar = 0;
      unsigned char* gdst = sm.G;
      for (int item = blockIdx.x; item < ar.nwork; item += gridDim.x) {
        const PulsarMeta pm = ar.meta[ar.pidx[item / ar.ntile]];
        const size_t stage_bytes = (size_t)V_STAGE + (size_t)NPL * pm.i8_rows * KT;
        const int ng = (pm.i8_rows + 127) >> 7;
        for (int grp = 0; grp < ng; ++grp) {  // one pass over the TOAs per group of 128 operand rows
          const int rows_g = min(128, pm.i8_rows - 128 * grp);
          const uint32_t gbytes = (uint32_t)(NPL * rows_g * KT);
          const unsigned char* src = ar.planes + pm.i8_off;
          const size_t goff = (size_t)V_STAGE + (size_t)grp * (NPL * 128 * KT);
          for (int c = 0; c < pm.i8_nst; ++c, ++k) {
            if (k >= VST) wait_wd<2000>(&sm.v_empty[sv], vpar ^ 1u, 1, k);
            mbar_expect_tx(&sm.v_full[sv], V_STAGE);
            tma_load_1d(sm.V + sv * V_STAGE, src, V_STAGE, &sm.v_full[sv]);
            if (k >= (uint32_t)ar.gst) wait_wd<2000>(&sm.g_empty[sg], gpar ^ 1u, 2, k);
            mbar_expect_tx(&sm.g_full[sg], gbytes);
            tma_load_1d(gdst, src + goff, gbytes, &sm.g_full[sg]);
            src += stage_bytes;
            if (++sv == VST) { sv = 0; vpar ^= 1u; }
            if (++sg == (uint32_t)ar.gst) { sg = 0; gpar ^= 1u; gdst = sm.G; } else gdst += ar.gslot;
          }
        }
      }
    }
  } else if (wid < 12) {
    // ================= consumer warpgroups: wgmma issue + epilogue, 64 operand rows each =================
    reg_alloc<REGS_CONS>();
    const int cwg = (wid - 4) >> 2;          // operand rows 64 cwg .. 64 cwg + 63 of the row group
    const int cw = (wid - 4) & 3;            // warp inside the warpgroup: 16 of those rows
    const int lr0 = 64 * cwg + 16 * cw + (lane >> 2);  // accumulator rows lr0 and lr0 + 8 of this thread
    const uint32_t g0 = smem_u32(sm.G), s0 = smem_u32(sm.S);
    uint32_t acc[NPL][NACC];
    uint32_t k = 0, it = 0;
    uint32_t sg = 0, gpar = 0, ss = 0, spar = 0, ga = g0, sa = s0;  // ring positions, parities, slot addresses
    for (int item = blockIdx.x; item < ar.nwork; item += gridDim.x, ++it) {
      const int gp = item / ar.ntile, ft = item - gp * ar.ntile;
      const int p = ar.pidx[gp];
      const PulsarMeta pm = ar.meta[p];
      const int64_t f0 = (int64_t)ft * NF;
      // bases wider than 127 columns take one pass per group of 128 operand rows; the b-sums of the groups add up in
      // `part`, the w row sits in the last group
      for (int grp = 0; 128 * grp < pm.i8_rows; ++grp) {
        const int rows_g = min(128, pm.i8_rows - 128 * grp);
        const bool active = 64 * cwg < rows_g;  // warpgroup-uniform: this warpgroup's rows exist in the group
        const uint32_t aplane16 = (uint32_t)(rows_g * KT) >> 4;
        uint32_t psg = 0, pss = 0;  // slots of the previous stage, released once its MMAs have completed
        for (int c = 0; c < pm.i8_nst; ++c, ++k) {
          wait_wd<0>(&sm.g_full[sg], gpar, 4, k);
          wait_wd<0>(&sm.s_full[ss], spar, 5, k);
          __syncwarp();  // lanes leave the polling loops independently; the .aligned wgmma instructions need them converged
          if (active) {
            wgmma_fence();
            issue_stage(acc, desc_lo(ga + (uint32_t)(64 * cwg * KT)), desc_lo(sa), aplane16, c == 0);
            wgmma_commit();
            wgmma_wait<1>();  // the stage before this one has been read
          }
          if (c > 0 && (tid & 127) == 0) { mbar_arrive(&sm.g_empty[psg]); mbar_arrive(&sm.s_empty[pss]); }
          psg = sg; pss = ss;
          if (++sg == (uint32_t)ar.gst) { sg = 0; gpar ^= 1u; ga = g0; } else ga += (uint32_t)ar.gslot;
          if (++ss == SST) { ss = 0; spar ^= 1u; sa = s0; } else sa += S_STAGE;
        }
        if (active) wgmma_wait<0>();
        if ((tid & 127) == 0) { mbar_arrive(&sm.g_empty[psg]); mbar_arrive(&sm.s_empty[pss]); }

        // ---- epilogue of the pass: thread holds rows lr0, lr0 + 8 x frequencies 8 jn + 2 (lane & 3) + e
        double v[4][3];  // per frequency slot q = 2 jn + e: the two rows' contributions to the three b-sums
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q][0] = v[q][1] = v[q][2] = 0.0;
        if (active) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = 128 * grp + lr0 + 8 * h;
            const double rs = ar.rowscale[(size_t)p * RS + row];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int jn = q >> 1, e = q & 1;
              const int is = 4 * jn + 2 * h + e, ic = is + 8;  // sin column 8 jn + .., cos column 16 + the same
              double ys = (double)(int)acc[NPL - 1][is], yc = (double)(int)acc[NPL - 1][ic];  // smallest weight first
#pragma unroll
              for (int g = NPL - 2; g >= 0; --g) {
                ys = fma(ys, 0.00390625, (double)(int)acc[g][is]);
                yc = fma(yc, 0.00390625, (double)(int)acc[g][ic]);
              }
              ys *= rs;
              yc *= rs;
              const int fl = 8 * jn + 2 * (lane & 3) + e;  // frequency inside the tile
              if (row == pm.m) {  // the w row: (s|r) = s.w, (c|r) = c.w  (DESIGN.md section 2)
                sm.nval[2 * fl] = ys;
                sm.nval[2 * fl + 1] = yc;
              }
              if (NMFP && row >= pm.mfix && row < pm.m && f0 + fl < ar.F) {
                // rows of the per-draw block leave as z'
                double* z = ar.nm.z(p, f0 + fl, ar.nt32, row - pm.mfix + (ar.nm.mvpad - pm.mvar));
                z[0] = ys;
                z[16] = yc;
              }
              if (row < pm.mfix) {  // rows of the draw-independent block enter the b-sums (plain Fp: all)
                v[q][0] = fma(ys, ys, v[q][0]);
                v[q][1] = fma(ys, yc, v[q][1]);
                v[q][2] = fma(yc, yc, v[q][2]);
              }
            }
          }
        }
        // sum over the 8 lanes that share (lane & 3): the 16 rows of this warp
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int k2 = 0; k2 < 3; ++k2) {
            double t = v[q][k2];
            t += __shfl_xor_sync(0xffffffffu, t, 4);
            t += __shfl_xor_sync(0xffffffffu, t, 8);
            t += __shfl_xor_sync(0xffffffffu, t, 16);
            v[q][k2] = t;
          }
        if (lane < 4) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int fl = 8 * (q >> 1) + 2 * lane + (q & 1);
            double* o = sm.part + ((size_t)(wid - 4) * NF + fl) * 3;
            if (grp == 0) { o[0] = v[q][0]; o[1] = v[q][1]; o[2] = v[q][2]; }
            else { o[0] += v[q][0]; o[1] += v[q][1]; o[2] += v[q][2]; }   // (this warp's own slots: no other writer)
          }
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");  // partial sums and the w-row values of the 8 warps are visible
      const uint32_t buf = it & 1u;
      if (wid == 4) {
        wait_wd<2000>(&sm.sums_full[buf], (it >> 1) & 1u, 7, it);
        if (lane < NF) {
          const int f = lane;
          const int64_t fidx = f0 + f;
          double b[3] = {0, 0, 0}, a[3];
#pragma unroll
          for (int w2 = 0; w2 < 8; ++w2)
#pragma unroll
            for (int k2 = 0; k2 < 3; ++k2) b[k2] += sm.part[((size_t)w2 * NF + f) * 3 + k2];
#pragma unroll
          for (int k2 = 0; k2 < 2; ++k2)
            a[k2] = sm.redA[((buf * 2 + 0) * NF + f) * 3 + k2] + sm.redA[((buf * 2 + 1) * NF + f) * 3 + k2];
          a[2] = pm.ninv_sum - a[0];  // c N^-1 c = sum 1/N - s N^-1 s (s^2 + c^2 = 1 to the last bit of the sincos values)
          const double N0 = sm.nval[2 * f], N1 = sm.nval[2 * f + 1];  // (s|r), (c|r)
          if (fidx < ar.F) {
            if (NMFP) ar.nm.put_a(p, fidx, ar.nt32, a[0] - b[0], a[1] - b[1], a[2] - b[2], N0, N1);
            else ar.fp.put(p, fidx, ar.F, ar.freqs[fidx], a[0] - b[0], a[1] - b[1], a[2] - b[2], N0, N1);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.sums_empty[buf]);
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");  // part / nval are rewritten by the next item
    }
  } else {
    // ================= producers: sin/cos digit planes + the two quadratic sums =================
    reg_dealloc<REGS_PROD>();
    const int pw = wid - 12;
    const uint32_t grp = (uint32_t)(pw >> 2);          // serves the stages with (global stage index % 2) == grp
    // lane = 4 * kg + fl: the 8 lanes of a quarter-warp read two distinct (t, 1/N) entries 64 bytes apart (no bank
    // conflict on the 16-byte loads), and a warp's 4-byte stores cover 4 rows x 32 bytes = all 32 banks
    const int kg = lane >> 2, fl = lane & 3;
    const int f = 4 * (pw & 3) + fl;                   // frequency inside the tile
    const int soff = swz32(f, 4 * kg);                 // word of TOAs 4kg..4kg+3 in row f (sin); cos row: + NF rows
    // A group announces stage k (s_full) after the fp64 part of its NEXT stage, so that the MMAs of stage k run next to
    // the integer part of stage k + 2 (digits, byte transpose, stores) rather than next to an fp64 part.
    auto store_planes = [&](const double (&sv4)[4], const double (&cv4)[4], unsigned char* sb) {
      uint32_t slo[4], shi[4], clo[4], chi[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const uint2 ds = digits7(sv4[e]), dc = digits7(cv4[e]);
        slo[e] = ds.x; shi[e] = ds.y; clo[e] = dc.x; chi[e] = dc.y;
      }
      // word of plane p (most significant first) = byte (6 - p) of the four values
      {
        const uint32_t a = __byte_perm(slo[0], slo[1], 0x5140), b = __byte_perm(slo[0], slo[1], 0x7362);
        const uint32_t c2 = __byte_perm(slo[2], slo[3], 0x5140), d = __byte_perm(slo[2], slo[3], 0x7362);
        const uint32_t e2 = __byte_perm(shi[0], shi[1], 0x5140), f2 = __byte_perm(shi[0], shi[1], 0x7362);
        const uint32_t g2 = __byte_perm(shi[2], shi[3], 0x5140), h2 = __byte_perm(shi[2], shi[3], 0x7362);
        *reinterpret_cast<uint32_t*>(sb + 6 * S_PLANE) = __byte_perm(a, c2, 0x5410);   // byte 0
        *reinterpret_cast<uint32_t*>(sb + 5 * S_PLANE) = __byte_perm(a, c2, 0x7632);   // byte 1
        *reinterpret_cast<uint32_t*>(sb + 4 * S_PLANE) = __byte_perm(b, d, 0x5410);    // byte 2
        *reinterpret_cast<uint32_t*>(sb + 3 * S_PLANE) = __byte_perm(b, d, 0x7632);    // byte 3
        *reinterpret_cast<uint32_t*>(sb + 2 * S_PLANE) = __byte_perm(e2, g2, 0x5410);  // byte 4
        *reinterpret_cast<uint32_t*>(sb + 1 * S_PLANE) = __byte_perm(e2, g2, 0x7632);  // byte 5
        *reinterpret_cast<uint32_t*>(sb + 0 * S_PLANE) = __byte_perm(f2, h2, 0x5410);  // byte 6
      }
      {
        unsigned char* cb = sb + NF * KT;  // cos rows NF..2NF-1
        const uint32_t a = __byte_perm(clo[0], clo[1], 0x5140), b = __byte_perm(clo[0], clo[1], 0x7362);
        const uint32_t c2 = __byte_perm(clo[2], clo[3], 0x5140), d = __byte_perm(clo[2], clo[3], 0x7362);
        const uint32_t e2 = __byte_perm(chi[0], chi[1], 0x5140), f2 = __byte_perm(chi[0], chi[1], 0x7362);
        const uint32_t g2 = __byte_perm(chi[2], chi[3], 0x5140), h2 = __byte_perm(chi[2], chi[3], 0x7362);
        *reinterpret_cast<uint32_t*>(cb + 6 * S_PLANE) = __byte_perm(a, c2, 0x5410);
        *reinterpret_cast<uint32_t*>(cb + 5 * S_PLANE) = __byte_perm(a, c2, 0x7632);
        *reinterpret_cast<uint32_t*>(cb + 4 * S_PLANE) = __byte_perm(b, d, 0x5410);
        *reinterpret_cast<uint32_t*>(cb + 3 * S_PLANE) = __byte_perm(b, d, 0x7632);
        *reinterpret_cast<uint32_t*>(cb + 2 * S_PLANE) = __byte_perm(e2, g2, 0x5410);
        *reinterpret_cast<uint32_t*>(cb + 1 * S_PLANE) = __byte_perm(e2, g2, 0x7632);
        *reinterpret_cast<uint32_t*>(cb + 0 * S_PLANE) = __byte_perm(f2, h2, 0x5410);
      }
    };
    uint32_t kbase = 0, it = 0;
    int pend = -1;  // S slot whose planes are stored but not announced yet
    for (int item = blockIdx.x; item < ar.nwork; item += gridDim.x, ++it) {
      const int gp = item / ar.ntile, ft = item - gp * ar.ntile;
      const PulsarMeta pm = ar.meta[ar.pidx[gp]];
      const int64_t f0 = (int64_t)ft * NF;
      const double fq = ar.freqs[f0 + f < ar.F ? f0 + f : f0];  // a short last tile repeats its first frequency
      const double omega = __dmul_rn(6.283185307179586, fq);     // (2*pi)*f, rounded once (fastfp.py:78)
      const bool fast = __all_sync(0xffffffffu, fabs(omega) * pm.tabs_max <= 0.999 * FFP_SINCOS_MAX);
      double s3[2] = {0.0, 0.0};  // s N^-1 s, s N^-1 c
      const int nst = pm.i8_nst;
      // one pass over the TOAs per group of 128 operand rows (bases wider than 127 columns): the planes are produced
      // again for every pass, the quadratic sums only in the first
      for (int rg = 0; 128 * rg < pm.i8_rows; ++rg, kbase += (uint32_t)nst) {
      const int c0 = (int)((kbase ^ grp) & 1u);
      for (int c = c0; c < nst; c += 2) {
        const uint32_t k = kbase + (uint32_t)c;
        const uint32_t sv = k % VST, ss = k % SST;
        wait_wd<2000>(&sm.v_full[sv], (k / VST) & 1u, 8, k);
        const double2* vv = reinterpret_cast<const double2*>(sm.V + sv * V_STAGE) + 4 * kg;
        // ---- fp64 part: four (TOA, frequency) pairs per thread
        double ph[4], ninv[4], sv4[4], cv4[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const double2 tn = vv[e];                    // (t, 1/N)
          ph[e] = __dmul_rn(omega, tn.x);              // ((2*pi)*f)*t, rounded once more
          ninv[e] = tn.y;
        }
        if (fast) {
          sincos_cw_n<4>(ph, sv4, cv4);  // in lockstep: phases inside the Cody-Waite range (checked once per item)
        } else {
          // cold: some phase of this item may exceed the Cody-Waite range (or is NaN/Inf): library sincos
#pragma unroll
          for (int e = 0; e < 4; ++e) {  // unrolled: a dynamic index would put the arrays in local memory
            double s1, c1;
            sincos(ph[e], &s1, &c1);
            sv4[e] = s1; cv4[e] = c1;
          }
        }
        if (rg == 0) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const double sn = sv4[e] * ninv[e];   // c N^-1 c follows from sum 1/N - s N^-1 s (epilogue)
            s3[0] = fma(sn, sv4[e], s3[0]);
            s3[1] = fma(sn, cv4[e], s3[1]);
          }
        }
        // ---- the group's previous stage is complete in shared memory: announce it now (see above)
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&sm.v_empty[sv]);
          if (pend >= 0) mbar_arrive(&sm.s_full[pend]);
        }
        // ---- integer part: digits, 4 x 7 byte transpose, stores
        if (k >= SST) wait_wd<2000>(&sm.s_empty[ss], ((k / SST) - 1) & 1u, 9, k);
        store_planes(sv4, cv4, sm.S + ss * S_STAGE + soff);
        fence_proxy_async();  // generic-proxy stores -> visible to the tensor core's (async proxy) operand reads
        pend = (int)ss;
      }
      }
      // the two sums of frequency f: over the 8 lanes that share it (lane bits 2..4), then published per group
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        double t = s3[q];
        t += __shfl_xor_sync(0xffffffffu, t, 4);
        t += __shfl_xor_sync(0xffffffffu, t, 8);
        t += __shfl_xor_sync(0xffffffffu, t, 16);
        s3[q] = t;
      }
      const uint32_t buf = it & 1u;
      if (it >= 2) wait_wd<2000>(&sm.sums_empty[buf], ((it >> 1) - 1) & 1u, 10, it);
      if (kg == 0) {
        double* o = sm.redA + ((buf * 2 + grp) * NF + f) * 3;
        o[0] = s3[0]; o[1] = s3[1];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.sums_full[buf]);
    }
    __syncwarp();
    if (lane == 0 && pend >= 0) mbar_arrive(&sm.s_full[pend]);  // the group's last stage of this CTA
  }
  __syncthreads();
}

// ---- measurement helper: the tensor path's own ceilings (fastfp_fp64_peak kinds 17 and 18) -----------------------
// Back-to-back s8 wgmmas from two warpgroups per CTA (128 operand rows), one CTA per SM, operands in the sweep
// kernel's SWIZZLE_32B planes: N = 256 (one accumulator) gives the INT8 tensor peak of the chip, N = 32 with the
// sweep's 28-product stage into 7 accumulators gives the rate this formulation can reach at most.
__device__ __forceinline__ void wgmma_i8_n256(uint32_t (&d)[128], uint64_t da, uint64_t db) {
#define R8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, 1;\n"
      : R8(0), R8(8), R8(16), R8(24), R8(32), R8(40), R8(48), R8(56), R8(64), R8(72), R8(80), R8(88), R8(96), R8(104),
        R8(112), R8(120)
      : "l"(da), "l"(db));
#undef R8
}

template <int N>
__global__ void __launch_bounds__(256, 1) i8_peak_kernel(int iters, int* out) {
  extern __shared__ __align__(1024) unsigned char smem[];
  constexpr int A_PLANE = 128 * KT, B_PLANE = N * KT;
  unsigned char* sA = smem;
  unsigned char* sB = smem + NPL * A_PLANE;
  for (int i = threadIdx.x; i < NPL * (A_PLANE + B_PLANE); i += blockDim.x) smem[i] = (unsigned char)((i * 7 + 3) & 3);
  fence_proxy_async();
  __syncthreads();
  const uint32_t a_lo = desc_lo(smem_u32(sA) + (uint32_t)((threadIdx.x >> 7) * 64 * KT)), b_lo = desc_lo(smem_u32(sB));
  uint32_t sum = 0;
  if (N == 256) {
    uint32_t d[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) d[i] = 0;
    wgmma_fence();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
      for (int i = 0; i < NPL; ++i)
#pragma unroll
        for (int j = 0; j < NPL - i; ++j)
          wgmma_i8_n256(d, DESC_HI | (uint64_t)(a_lo + (uint32_t)(i * A_PLANE / 16)),
                        DESC_HI | (uint64_t)(b_lo + (uint32_t)(j * B_PLANE / 16)));
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 128; ++i) sum += d[i];
  } else {
    uint32_t acc[NPL][NACC];
    wgmma_fence();
    for (int it = 0; it < iters; ++it) {
      issue_stage(acc, a_lo, b_lo, A_PLANE / 16, it == 0);
      wgmma_commit();
      wgmma_wait<1>();
    }
    wgmma_wait<0>();
#pragma unroll
    for (int g = 0; g < NPL; ++g)
#pragma unroll
      for (int i = 0; i < NACC; ++i) sum += acc[g][i];
  }
  if (out) out[blockIdx.x * blockDim.x + threadIdx.x] = (int)sum;
}

}  // namespace i8

int run_i8_peak(int kind, int iters, double* tops, double* ms_out) {
  using namespace i8;
  int dev = 0, sms = 0;
  FFP_CUDA(cudaGetDevice(&dev));
  FFP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int N = kind == 17 ? 256 : 32;
  const size_t smem = (size_t)NPL * (128 + N) * KT + 1024;
  if (kind == 17) FFP_CUDA(cudaFuncSetAttribute(i8_peak_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  else FFP_CUDA(cudaFuncSetAttribute(i8_peak_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  Event e0, e1;
  FFP_CUDA(event_create(&e0));
  FFP_CUDA(event_create(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {
    FFP_CUDA(cudaEventRecord(e0.get()));
    if (kind == 17) i8_peak_kernel<256><<<sms, 256, smem>>>(iters, nullptr);
    else i8_peak_kernel<32><<<sms, 256, smem>>>(iters, nullptr);
    FFP_CUDA(cudaEventRecord(e1.get()));
    FFP_CUDA(cudaEventSynchronize(e1.get()));
    float ms = 0;
    FFP_CUDA(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
    if (rep > 0 && ms < best) best = ms;
  }
  g_launches += 4;
  FFP_CUDA(cudaGetLastError());
  *tops = 2.0 * (double)sms * iters * 28.0 * 128.0 * N * 32.0 / (best * 1e-3) / 1e12;
  *ms_out = best;
  return 0;
}

// ---- host side ------------------------------------------------------------------------------------------------
// A pack can take the tensor path when every pulsar fits the tile: diagonal N, m + 1 <= 128 rows (the basis rows and
// the w row), n <= 16384 TOAs (int32 accumulators: 7 products of |digit|^2 <= 2^14 per TOA stay below 2^31
// up to 18 724 TOAs).
// which pulsars the tensor sweep can take: diagonal N (pack-wide), up to RS operand rows, n <= 16384 (exactness of the
// int32 accumulators); the others of a pack stay on the fp64 kernel in the same sweep
static bool i8_takes(const fastfp_pack* pk, const PulsarMeta& pm) {
  return !pk->ecorr && pm.m + 1 <= i8::RS && pm.n <= 16384;
}
bool i8_eligible(const fastfp_pack* pk) {
  for (const PulsarMeta& pm : pk->meta)
    if (i8_takes(pk, pm)) return true;
  return false;
}

// lay out and build the digit planes from the fp64 packets (after launch_fp_precompute) into pk->i8, which stays empty
// when no pulsar can take them
int build_i8_planes(fastfp_pack* pk, cudaStream_t st) {
  if (!i8_eligible(pk)) return 0;
  const int P = pk->P;
  int64_t off = 0;
  int rows_max = 0, nst_max = 0;
  for (PulsarMeta& pm : pk->meta) {
    pm.i8_rows = pm.i8_nst = 0;
    pm.i8_off = off;
    if (!i8_takes(pk, pm)) continue;
    // rows (basis + the w row; more than 128 of them form row groups, one pass over the TOAs each) padded to 32:
    // every plane then starts on a 1024-byte boundary of the (1024-aligned) ring, the alignment
    // the operand descriptors of all swizzle modes accept; rows beyond the padding are never loaded (the MMA reads
    // 128 rows per plane, the tail comes from the next plane and lands in output lanes nobody reads)
    pm.i8_rows = (pm.m + 1 + 31) / 32 * 32;
    pm.i8_nst = (pm.n + i8::KT - 1) / i8::KT;
    off += (int64_t)pm.i8_nst * (i8::V_STAGE + i8::NPL * pm.i8_rows * i8::KT);
    rows_max = pm.i8_rows > rows_max ? pm.i8_rows : rows_max;
    nst_max = pm.i8_nst > nst_max ? pm.i8_nst : nst_max;
  }
  const PackCore& c = pk->core;
  FFP_CUDA(cudaMemcpyAsync(c.meta.get(), pk->meta.data(), sizeof(PulsarMeta) * P, cudaMemcpyHostToDevice, st));
  TensorPath tp;
  // the last plane of the last stage is read 128 rows deep by the MMA only from shared memory; the global buffer
  // needs no slack, but keep the allocation 16-byte granular for the bulk copies
  FFP_CUDA(dev_alloc(&tp.planes, (size_t)off + 16));
  FFP_CUDA(dev_alloc(&tp.scale, (size_t)P * i8::RS));
  FFP_CUDA(cudaMemsetAsync(tp.scale.get(), 0, (size_t)P * i8::RS * sizeof(double), st));
  DeviceBuf<int> d_exp, d_bad;
  FFP_CUDA(dev_alloc(&d_exp, (size_t)P * i8::RS));
  FFP_CUDA(dev_alloc(&d_bad, (size_t)P));
  FFP_CUDA(cudaMemsetAsync(d_bad.get(), 0, (size_t)P * sizeof(int), st));
  i8::i8_rowscale_kernel<<<dim3(rows_max, P), 256, 0, st>>>(c.packets.get(), c.meta.get(), tp.scale.get(),
                                                            d_exp.get(), d_bad.get());
  i8::i8_planes_kernel<<<dim3(nst_max, P), 256, 0, st>>>(c.packets.get(), c.meta.get(), d_exp.get(),
                                                         tp.planes.get());
  g_launches += 2;
  cudaError_t e = cudaGetLastError();
  std::vector<int> bad(P, 0);
  if (e == cudaSuccess) e = cudaMemcpyAsync(bad.data(), d_bad.get(), (size_t)P * sizeof(int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return cuda_fail(e, "build_i8_planes");
  // pulsars with a non-finite G or w (singular Sigma, NaN data) cannot be carried by integer planes: fp64 kernel
  std::vector<int> take, rest_flag(P + pk->items.size(), 1);  // row-group items (wide pulsars) stay on the fp64 kernel
  for (int p = 0; p < P; ++p) {
    const bool ok = pk->meta[p].i8_nst > 0 && bad[p] == 0 && (p >= (int)pk->info.size() || pk->info[p] == 0);
    if (ok) { take.push_back(p); rest_flag[p] = 0; }
  }
  if (take.empty()) return 0;
  FFP_CUDA(dev_alloc(&tp.pidx, take.size()));
  FFP_CUDA(cudaMemcpy(tp.pidx.get(), take.data(), sizeof(int) * take.size(), cudaMemcpyHostToDevice));
  tp.count = (int)take.size();
  // the complement, per kernel family of the fp64 sweep
  for (Group& g : pk->groups) {
    std::vector<int> all((size_t)g.count), rest;
    FFP_CUDA(cudaMemcpy(all.data(), g.pidx.get(), sizeof(int) * g.count, cudaMemcpyDeviceToHost));
    for (int p : all)
      if (rest_flag[p]) rest.push_back(p);
    g.count_rest = (int)rest.size();
    if (g.count_rest) {
      FFP_CUDA(dev_alloc(&g.pidx_rest, rest.size()));
      FFP_CUDA(cudaMemcpy(g.pidx_rest.get(), rest.data(), sizeof(int) * rest.size(), cudaMemcpyHostToDevice));
    }
  }
  pk->bytes += off + (int64_t)P * i8::RS * 8;
  tp.rows_max = rows_max;
  tp.ok = true;
  pk->i8 = std::move(tp);
  return 0;
}

// one of fp, nm is set
static int launch_i8(const fastfp_pack* pk, const double* d_freqs, int64_t F, const FpOut* fp, const NmfpTiles* nm,
                     cudaStream_t st) {
  using namespace i8;
  Args a{};
  a.freqs = d_freqs;
  a.F = F;
  if (fp) a.fp = *fp;
  if (nm) a.nm = *nm;
  a.planes = pk->i8.planes.get();
  a.rowscale = pk->i8.scale.get();
  a.meta = pk->core.meta.get();
  a.pidx = pk->i8.pidx.get();
  const int64_t ntile = (a.F + NF - 1) / NF, nwork = ntile * pk->i8.count;  // the pulsars this kernel takes
  if (nwork > 0x7fffffffLL) { set_error("frequency batch too large for one launch"); return -1; }
  a.ntile = (int)ntile;
  a.nwork = (int)nwork;
  a.nt32 = (int)((a.F + 31) / 32);
  a.gslot = NPL * (pk->i8.rows_max < 128 ? pk->i8.rows_max : 128) * KT;  // one row group
  const size_t budget = 220 * 1024 - SMEM_FIXED;
  int gst = (int)(budget / a.gslot);
  gst = gst > 8 ? 8 : gst;
  // the last plane of the last slot is read 64 rows deep per warpgroup: the S ring behind the G ring absorbs the overrun
  if (gst < 2) { set_error("internal: no room for the G ring"); return FASTFP_ERR_UNSUPPORTED; }
  a.gst = gst;
  const size_t smem = (size_t)gst * a.gslot + SMEM_FIXED;
  static bool attr_done[64] = {};
  if (!attr_done[pk->device & 63]) {
    FFP_CUDA(cudaFuncSetAttribute(fp_sweep_i8_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    FFP_CUDA(cudaFuncSetAttribute(fp_sweep_i8_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_done[pk->device & 63] = true;
  }
  const unsigned grid = (unsigned)(nwork < pk->num_sms ? nwork : pk->num_sms);
  if (nm) fp_sweep_i8_kernel<true><<<grid, THREADS, smem, st>>>(a);
  else fp_sweep_i8_kernel<false><<<grid, THREADS, smem, st>>>(a);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

int launch_fp_sweep_i8(const fastfp_pack* pk, const double* d_freqs, int64_t F, const FpOut& out, cudaStream_t st) {
  return launch_i8(pk, d_freqs, F, &out, nullptr, st);
}
int launch_fp_sweep_i8(const fastfp_pack* pk, const double* d_freqs, int64_t F, const NmfpTiles& out,
                       cudaStream_t st) {
  return launch_i8(pk, d_freqs, F, nullptr, &out, st);
}

}  // namespace ffp
