// The frequency-sweep kernel (fp64 DMMA formulation): a persistent, warp-specialised CTA -- SweepCfg::NWC
// consumer (MMA) warps + SweepCfg::NWP producer (sincos) warps, 8 + 16 = 768 threads by default and 8 + 8 = 512
// for m <= 80, one CTA per SM -- takes (pulsar, frequency-tile) work items from an atomic counter.
//
// Replaces the body of FastFp.calculate_Fp under jax.vmap (reference fastfp/fastfp.py:69-92,
// examples/run_fp.py:63) -- and, in SweepMode::Nmfp, the draw-independent part of
// NMFP.calculate_nmfp (fastfp/nmfp.py:96-119) -- for a whole frequency tile at once:
//
//   per chunk of CI TOAs
//     TMA        : two bulk copies per chunk -- the TOA vectors (t, 1/N, w) (to the producers) and
//                  the G tile in MMA-fragment order (to the consumers) -- through mbarrier rings
//     producers  : build sin/cos of ((2*pi)*f)*t (fastfp.py:78-79 phase order, one rounding per
//                  multiply) for their (frequency, TOA) pairs, store them into the shared S-tile
//                  ring in MMA-fragment order, and accumulate s N^-1 s, s N^-1 c, c N^-1 c, s.w, c.w
//     consumers  : Y^T[2*KF][MP] += S_chunk^T . G_chunk on the fp64 MMA path (mma.sync.m16n8k4.f64: 16 rows =
//                  8 frequencies x {sin, cos}, 8 columns = basis rows, k = TOAs; it shares the pipe with DFMA
//                  but runs at twice m8n8k4's rate on H100, DESIGN.md section 4.1)
//   epilogue     : b = Y_s.Y_s, Y_s.Y_c, Y_c.Y_c; M = [[sNs-b_ss, sNc-b_sc],[.., cNc-b_cc]],
//                  N = [s.w, c.w]; general 2x2 solve with partial pivoting (what jnp.linalg.solve
//                  does at fastfp.py:90); term = 0.5 * N . M^-1 N.
//
// Producers and consumers are decoupled by full/empty mbarriers, so the dependent sincos chains of
// the producers interleave with the consumers' MMAs on the shared fp64 pipe at run time. The producers' DFMAs queue
// behind the MMAs on the shared pipe, so a sub-partition needs several independent sincos chains in flight to keep
// the S ring full: with the default split it hosts two consumer warps and four producer warps of one chain each
// (setmaxnreg split SweepCfg::CREGS / PREGS = 120 / 56 of the 768 x 80 pool); the m <= 80 family hosts two and two,
// whose producers run four chains in lockstep (168 / 88 of the 512 x 128 pool, which also keeps the consumers'
// accumulators and fragments out of local memory).
//
// The f^(-1/3) prefactor of fastfp.py:78-79 scales N by a and M by a^2 and cancels exactly in
// N^T M^-1 N; it is not applied (f <= 0 still yields NaN as in the reference).
//
// Summation is blocked: level-1 register sums over FLUSH_TOAS TOAs are folded into level-2
// totals that live in an L2-resident scratch slab (one per resident CTA), so the rounding error
// of the n-long sums stays at the level of a BLAS/XLA dot, and the register file holds only one
// set of accumulators.
#pragma once
#include "ffp_internal.cuh"
#include "ffp_sincos.cuh"

namespace ffp {

enum class SweepMode { Fp, Nmfp, Res };  // which output block the kernel writes

struct SweepArgs {
  const double* packets;
  const PulsarMeta* meta;
  const int* pidx;
  int ntile_f;
  int nwork;
  const double* freqs;
  int64_t F;
  // the output block of the kernel's mode (the realisations of SweepMode::Res are rows roundup8(m) .. roundup8(m)+R-1
  // of G). A union, since a kernel writes one: a parameter block of more than 128 bytes is read through a pointer
  // instead of straight from the constant bank, which changes the code of the whole kernel.
  union {
    FpOut fp;
    NmfpTiles nm;
    ResOut res;
  };
  RowGroupOut rg;         // SweepMode::Fp: the outputs of row-group items (DESIGN.md section 5h)
  double* slab;           // level-2 scratch, SLAB doubles per CTA
  unsigned int* counter;  // work counter (zeroed before the launch)
  const unsigned char* done_mask;  // block-N packs: per chunk, which of the 8 epoch slots end there
#ifdef FFP_DEBUG_SWITCHES
  int dbg;  // profiling builds only (tools/dbg_split.sh): bit 0 producers' math off, 1 MMAs off, 2 level-2 flush off
#endif
};
// The shipped library has no run-time switch that could skip work: the bits are a compile-time zero.
#ifdef FFP_DEBUG_SWITCHES
#define FFP_DBG(ar, bit) ((ar).dbg & (bit))
#else
#define FFP_DBG(ar, bit) 0
#endif

// Shared-memory carve-up, identical for both roles.
template <class C>
struct SweepSmem {
  double* Sring;   // [C::SST][KB][NX][32][2]  sin/cos tiles, A-fragment order (one (sin, cos) pair per lane)
  double* Gring;   // [GST][KB][NMB][32]      G tiles, B-fragment order
  double* Vring;   // [VST][VEC]           t | 1/N | w
  double* fq;      // [KF]                 trial frequencies of the current tile
  double* red;     // [RED]                epilogue reduction scratch
  uint64_t *s_full, *s_empty, *g_full, *g_empty, *v_full, *v_empty;
  __device__ explicit SweepSmem(unsigned char* raw) {
    Sring = reinterpret_cast<double*>(raw);
    Gring = Sring + C::SST * C::ST;
    Vring = Gring + C::GST * C::GT;
    fq = Vring + VST * C::VEC;
    red = fq + C::KF;
    s_full = reinterpret_cast<uint64_t*>(red + C::RED);
    s_empty = s_full + C::SST;
    g_full = s_empty + C::SST;
    g_empty = g_full + C::GST;
    v_full = g_empty + C::GST;
    v_empty = v_full + VST;
  }
};

struct WorkItem {
  int p, ft, nch;
  const double* gpk;
};

// ---- producer role: sin/cos tiles + the five weighted sums -----------------------------------
template <class C>
__device__ __forceinline__ void producer_loop(const SweepArgs& ar, SweepSmem<C>& sm, volatile int* s_work,
                                              const int pw, const int lane) {
  constexpr int XW = C::XW, SPW = C::SPW, KBW = C::KBW, NV = C::NV;
  const int tidp = pw * 32 + lane;
  const int bk = lane & 3, bf8 = lane >> 2;
  const int bx0 = C::NX >= C::NWP ? pw * XW : pw % C::NX;          // first group of 8 frequencies
  const int bsplit = C::NX >= C::NWP ? 0 : (pw / C::NX) * SPW;    // first partial sum; its k-blocks from bsplit*KBW
  // element (frequency group x, k-block kb) -> S offset (kb*NX + x)*64 + 2*lane: the (sin, cos) pair of a (TOA,
  // frequency) is the (a0, a1) fragment of the consumer lane with the same (frequency, TOA) -- one 16-byte store,
  // 512 contiguous bytes per warp
  const int sofs = 2 * lane;
  double* const sl = ar.slab + (size_t)blockIdx.x * C::SLAB + (size_t)C::NACCX * C::NTC + tidp;
  uint32_t g = 0;
  for (;;) {
    __syncthreads();  // B1: work item published
    const int w = *s_work;
    if (w >= ar.nwork) break;
    const int gp = w / ar.ntile_f;
    const PulsarMeta pm = ar.meta[ar.pidx[gp]];
    const double* gpk = ar.packets + pm.pk_off;
    const int nch = pm.nch;
    auto issue_vec = [&](int c) {
      const uint32_t k = g + (uint32_t)c;
      uint64_t* b = &sm.v_full[k % VST];
      mbar_expect_tx(b, C::VEC * 8);
      tma_load_1d(sm.Vring + (k % VST) * C::VEC, gpk + (size_t)c * C::PK, C::VEC * 8, b);
    };
    if (pw == 0 && lane == 0)
      for (int c = 0; c < VST - 1 && c < nch; ++c) issue_vec(c);
    __syncthreads();  // B2: frequencies of the tile are in shared memory
    double omega[XW];
#pragma unroll
    for (int xx = 0; xx < XW; ++xx)
      omega[xx] = __dmul_rn(6.283185307179586, sm.fq[8 * (bx0 + xx) + bf8]);  // (2*pi)*f, rounded once
    bool fast = true;  // warp-uniform in practice; any lane out of range sends its warp down the cold path
#pragma unroll
    for (int xx = 0; xx < XW; ++xx) fast = fast && (fabs(omega[xx]) * pm.tabs_max <= 0.999 * FFP_SINCOS_MAX);
    fast = __all_sync(0xffffffffu, fast);
    double s2[SPW][XW][5];  // [partial sum][frequency group][sum]
#pragma unroll
    for (int sp = 0; sp < SPW; ++sp)
#pragma unroll
      for (int xx = 0; xx < XW; ++xx)
#pragma unroll
        for (int q = 0; q < 5; ++q) s2[sp][xx][q] = 0.0;
    bool flushed = false;

    for (int c = 0; c < nch; ++c) {
      const uint32_t k = g + (uint32_t)c;
      if (pw == 0 && lane == 0 && c + VST - 2 < nch && c >= 1) {
        if (k >= 2) mbar_wait(&sm.v_empty[(k - 2) % VST], ((k - 2) / VST) & 1u);
        issue_vec(c + VST - 2);
      }
      mbar_wait(&sm.v_full[k % VST], (k / VST) & 1u);
      if (k >= C::SST) mbar_wait(&sm.s_empty[k % C::SST], ((k / C::SST) - 1) & 1u);
      const double* pk = sm.Vring + (k % VST) * C::VEC;
      double* sb = sm.Sring + (k % C::SST) * C::ST + sofs;
      if (!FFP_DBG(ar, 1) && pw < C::NACTIVE) {
#pragma unroll
        for (int sp = 0; sp < SPW; ++sp) {
          // element e of partial sum sp: k-block (bsplit + sp)*KBW + e/XW, frequency group bx0 + e%XW
          const int kb0 = (bsplit + sp) * KBW;
          if (fast) {
            // straight-line: every phase of this tile is inside the Cody-Waite range (checked once per
            // work item against the pulsar's largest |TOA|), so there is no per-element test; NV elements
            // at a time, whose sincos chains run in lockstep
#pragma unroll
            for (int e0 = 0; e0 < KBW * XW; e0 += NV) {
              double ph[NV], s[NV], cs[NV], ni[NV], wv[NV];
#pragma unroll
              for (int v = 0; v < NV; ++v) {
                const int i = 4 * (kb0 + (e0 + v) / XW) + bk;
                const double2 tn = *reinterpret_cast<const double2*>(pk + 4 * i);  // (t, 1/N)
                ph[v] = __dmul_rn(omega[(e0 + v) % XW], tn.x);  // ((2*pi)*f)*t, rounded once more
                ni[v] = tn.y;
                wv[v] = pk[4 * i + 2];
              }
              sincos_cw_n<NV>(ph, s, cs);
#pragma unroll
              for (int v = 0; v < NV; ++v) {
                const int kb = kb0 + (e0 + v) / XW, xx = (e0 + v) % XW;
                *reinterpret_cast<double2*>(sb + (kb * C::NX + bx0 + xx) * 64) = make_double2(s[v], cs[v]);
                const double sn = s[v] * ni[v], cn = cs[v] * ni[v];
                double* a = s2[sp][xx];
                a[0] = fma(sn, s[v], a[0]);
                a[1] = fma(sn, cs[v], a[1]);
                a[2] = fma(cn, cs[v], a[2]);
                a[3] = fma(s[v], wv[v], a[3]);
                a[4] = fma(cs[v], wv[v], a[4]);
              }
            }
          } else {
            // cold: some phase of this tile may exceed the Cody-Waite range (or is NaN/Inf): library sincos
#pragma unroll 1
            for (int e = 0; e < KBW * XW; ++e) {
              const int kb = kb0 + e / XW, xx = e % XW;
              const int i = 4 * kb + bk;
              const double om = __dmul_rn(6.283185307179586, sm.fq[8 * (bx0 + xx) + bf8]);
              const double ph = __dmul_rn(om, pk[4 * i]);
              double s, cs;
              sincos(ph, &s, &cs);
              const double ni = pk[4 * i + 1], wv = pk[4 * i + 2];
              *reinterpret_cast<double2*>(sb + (kb * C::NX + bx0 + xx) * 64) = make_double2(s, cs);
              const double sn = s * ni, cn = cs * ni;
#pragma unroll
              for (int x2 = 0; x2 < XW; ++x2)
                if (x2 == xx) {
                  s2[sp][x2][0] = fma(sn, s, s2[sp][x2][0]);
                  s2[sp][x2][1] = fma(sn, cs, s2[sp][x2][1]);
                  s2[sp][x2][2] = fma(cn, cs, s2[sp][x2][2]);
                  s2[sp][x2][3] = fma(s, wv, s2[sp][x2][3]);
                  s2[sp][x2][4] = fma(cs, wv, s2[sp][x2][4]);
                }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&sm.s_full[k % C::SST]);
        mbar_arrive(&sm.v_empty[k % VST]);
      }
      if ((c + 1) % C::FLUSH == 0 && c + 1 < nch && !FFP_DBG(ar, 4)) {
#pragma unroll
        for (int sp = 0; sp < SPW; ++sp)
#pragma unroll
          for (int xx = 0; xx < XW; ++xx)
#pragma unroll
            for (int q = 0; q < 5; ++q) {
              double* a = sl + (size_t)((sp * XW + xx) * 5 + q) * C::NTP;
              if (flushed) atomicAdd(a, s2[sp][xx][q]);  // result unused -> RED.ADD.F64, no round trip
              else __stcg(a, s2[sp][xx][q]);
              s2[sp][xx][q] = 0.0;
            }
        flushed = true;
      }
    }
    g += (uint32_t)nch;
    // scalar sums: level-2 totals, then across the 4 lanes that share a frequency
    if (flushed) __threadfence();
#pragma unroll
    for (int sp = 0; sp < SPW; ++sp)
#pragma unroll
      for (int xx = 0; xx < XW; ++xx)
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          double v = s2[sp][xx][q];
          if (flushed) v += __ldcg(sl + (size_t)((sp * XW + xx) * 5 + q) * C::NTP);
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          s2[sp][xx][q] = v;
        }
    double* redA = sm.red + C::WMW * C::KF * 3;  // [KSPLIT][KF][5]
    if (bk == 0 && pw < C::NACTIVE) {
#pragma unroll
      for (int sp = 0; sp < SPW; ++sp)
#pragma unroll
        for (int xx = 0; xx < XW; ++xx)
#pragma unroll
          for (int q = 0; q < 5; ++q)
            redA[((bsplit + sp) * C::KF + 8 * (bx0 + xx) + bf8) * 5 + q] = s2[sp][xx][q];
    }
    __syncthreads();  // B3: reductions published
    __syncthreads();  // B4: tile finished
  }
}

// Residual batches (DESIGN.md section 5d): rows from roundup8(m) on hold w_k = C^-1 r_k, so Y there is ((s|r_k),
// (c|r_k)); one 2x2 system per (realisation, frequency) with the M of the frequency, which redB[fl][3] holds. With a
// block-diagonal N, w_k already carries the whole N^-1, so these rows need no epoch fold; the slot rows sit at mpad - 8,
// after every realisation row read here.
// acc[r][q]: as in consumer_loop's epilogue.
template <class C>
__device__ __forceinline__ void res_tail(const ResOut& out, int64_t F, const SweepSmem<C>& sm,
                                         const double (&acc)[C::NMBW][C::NNB / 2][4], const double* redB, int p,
                                         int64_t f0, int m, int wm, int wn, int lane) {
  constexpr int NMBW = C::NMBW, NMT = C::NNB / 2;
  asm volatile("bar.sync 1, %0;" ::"n"(C::NTC) : "memory");  // consumers only: M of every frequency is published
  const int r0 = (m + 7) & ~7;
#pragma unroll
  for (int q = 0; q < NMT; ++q) {
    const int fl = 8 * (wn * NMT + q) + (lane >> 2);
    const int64_t f = f0 + fl;
    if (f >= F) continue;
    const double m00 = redB[fl * 3], m01 = redB[fl * 3 + 1], m11 = redB[fl * 3 + 2], fq = sm.fq[fl];
#pragma unroll
    for (int r = 0; r < NMBW; ++r)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int k = 8 * (wm * NMBW + r) + 2 * (lane & 3) + e - r0;
      if (k < 0 || k >= out.R) continue;
      out.put(k, p, f, F, fq, m00, m01, m11, acc[r][q][e], acc[r][q][2 + e]);
    }
  }
}

// ---- consumer role: the contraction and the epilogue -----------------------------------------
template <class C, SweepMode MODE, bool ECORR>
__device__ __forceinline__ void consumer_loop(const SweepArgs& ar, SweepSmem<C>& sm, volatile int* s_work,
                                              const int cw, const int lane) {
  // a warp owns NMBW blocks of 8 basis rows (the N side, B = G^T) x NMT tiles of 8 frequencies x {sin, cos} (the M
  // side, A = S^T): lane (g, t) = (lane>>2, lane&3) loads sin and cos of (frequency g, TOA t) as one 16-byte pair
  constexpr int NMBW = C::NMBW, NMT = C::NNB / 2;
  static_assert(C::NNB % 2 == 0, "16-row MMA tiles: frequencies in groups of 8");
  const int tid = cw * 32 + lane;
  const int wm = cw / C::WNW, wn = cw - wm * C::WNW;
  double* const sl = ar.slab + (size_t)blockIdx.x * C::SLAB + tid;
  uint32_t g = 0;
  for (;;) {
    if (tid == 0) *s_work = (int)atomicAdd(ar.counter, 1u);
    __syncthreads();  // B1
    const int w = *s_work;
    if (w >= ar.nwork) break;
    const int gp = w / ar.ntile_f, ft = w - gp * ar.ntile_f;
    const int p = ar.pidx[gp];
    const PulsarMeta pm = ar.meta[p];
    const double* gpk = ar.packets + pm.pk_off;
    const int nch = pm.nch;
    const int64_t f0 = (int64_t)ft * C::KF;
    auto issue_G = [&](int c) {
      const uint32_t k = g + (uint32_t)c;
      uint64_t* b = &sm.g_full[k % C::GST];
      mbar_expect_tx(b, C::GT * 8);
      tma_load_1d(sm.Gring + (k % C::GST) * C::GT, gpk + (size_t)c * C::PK + C::VEC, C::GT * 8, b);
    };
    if (tid == 0)
      for (int c = 0; c < C::GST - 1 && c < nch; ++c) issue_G(c);  // chunks 0 .. GST-2 in flight
    // a short last tile repeats its first frequency, so which sincos path a warp takes (and with it the last bits of
    // a bin) never depends on how many bins were passed along with it
    if (tid < C::KF) sm.fq[tid] = ar.freqs[f0 + tid < ar.F ? f0 + tid : f0];
    __syncthreads();  // B2

    // acc[r][q]: Y_sin of frequency 8*(wn*NMT + q) + g for basis rows 8*(wm*NMBW + r) + 2t + {0, 1}, then Y_cos
    double acc[NMBW][NMT][4];
#pragma unroll
    for (int r = 0; r < NMBW; ++r)
#pragma unroll
      for (int q = 0; q < NMT; ++q) acc[r][q][0] = acc[r][q][1] = acc[r][q][2] = acc[r][q][3] = 0.0;
    bool flushed = false;
    // block-diagonal N (kernel ECORR): the last row block of the last warp row holds 8 epoch slots (this thread:
    // slots 2t, 2t+1, kept apart); Y there is sqrt(beta_e) * sum_{i in e} x_i / N_i, folded into these sums when the
    // epoch ends
    double es[NMT][2][3];
#pragma unroll
    for (int q = 0; q < NMT; ++q)
#pragma unroll
      for (int e = 0; e < 2; ++e) es[q][e][0] = es[q][e][1] = es[q][e][2] = 0.0;
    const bool slot_warp = ECORR && wm == C::WMW - 1;
    const unsigned char* dmask = ECORR ? ar.done_mask + pm.dm_off : nullptr;

    // fragments of the next k-block -- also across chunk boundaries -- are fetched while the MMAs of
    // the current one run
    double2 a0[NMT];
    double b0[NMBW];
    {
      const uint32_t k = g;
      mbar_wait_spin(&sm.g_full[k % C::GST], (k / C::GST) & 1u);
      mbar_wait_spin(&sm.s_full[k % C::SST], (k / C::SST) & 1u);
      const double* gt = sm.Gring + (k % C::GST) * C::GT + (wm * NMBW) * 32 + lane;
      const double* sb = sm.Sring + (k % C::SST) * C::ST + (wn * NMT) * 64 + 2 * lane;
#pragma unroll
      for (int r = 0; r < NMBW; ++r) b0[r] = gt[r * 32];
#pragma unroll
      for (int q = 0; q < NMT; ++q) a0[q] = *reinterpret_cast<const double2*>(sb + q * 64);
    }
    for (int c = 0; c < nch; ++c) {
      const uint32_t k = g + (uint32_t)c;
      // the issuer refills the stage freed two chunks ago, so its wait practically never blocks
      if (tid == 0 && c + C::GST - 2 < nch && c >= 1) {
        if (k >= 2) mbar_wait(&sm.g_empty[(k - 2) % C::GST], ((k - 2) / C::GST) & 1u);
        issue_G(c + C::GST - 2);
      }
      const double* gt = sm.Gring + (k % C::GST) * C::GT + (wm * NMBW) * 32 + lane;
      const double* sb = sm.Sring + (k % C::SST) * C::ST + (wn * NMT) * 64 + 2 * lane;
#pragma unroll
      for (int kb = 0; kb < C::KB; ++kb) {
        double2 a1[NMT];
        double b1[NMBW];
        if (kb + 1 < C::KB) {
#pragma unroll
          for (int r = 0; r < NMBW; ++r) b1[r] = gt[((kb + 1) * C::NMB + r) * 32];
#pragma unroll
          for (int q = 0; q < NMT; ++q) a1[q] = *reinterpret_cast<const double2*>(sb + ((kb + 1) * C::NX + q) * 64);
        } else if (c + 1 < nch) {
          const uint32_t k1 = k + 1;
          mbar_wait_spin(&sm.g_full[k1 % C::GST], (k1 / C::GST) & 1u);
          mbar_wait_spin(&sm.s_full[k1 % C::SST], (k1 / C::SST) & 1u);
          const double* gt1 = sm.Gring + (k1 % C::GST) * C::GT + (wm * NMBW) * 32 + lane;
          const double* sb1 = sm.Sring + (k1 % C::SST) * C::ST + (wn * NMT) * 64 + 2 * lane;
#pragma unroll
          for (int r = 0; r < NMBW; ++r) b1[r] = gt1[r * 32];
#pragma unroll
          for (int q = 0; q < NMT; ++q) a1[q] = *reinterpret_cast<const double2*>(sb1 + q * 64);
        } else {
#pragma unroll
          for (int r = 0; r < NMBW; ++r) b1[r] = 0.0;
#pragma unroll
          for (int q = 0; q < NMT; ++q) a1[q] = make_double2(0.0, 0.0);
        }
        if (!FFP_DBG(ar, 2)) {
#pragma unroll
          for (int r = 0; r < NMBW; ++r)
#pragma unroll
            for (int q = 0; q < NMT; ++q) dmma_m16n8k4(acc[r][q], a0[q].x, a0[q].y, b0[r]);
        }
#pragma unroll
        for (int r = 0; r < NMBW; ++r) b0[r] = b1[r];
#pragma unroll
        for (int q = 0; q < NMT; ++q) a0[q] = a1[q];
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&sm.g_empty[k % C::GST]);
        mbar_arrive(&sm.s_empty[k % C::SST]);
      }
      if (ECORR && slot_warp) {
        // epochs that end in this chunk: e_xy += (sqrt(beta) A_x)(sqrt(beta) A_y); the slot restarts
        const unsigned dm = (unsigned)dmask[c] >> (2 * (lane & 3));
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if ((dm >> e) & 1u) {
#pragma unroll
            for (int q = 0; q < NMT; ++q) {
              const double ys = acc[NMBW - 1][q][e], yc = acc[NMBW - 1][q][2 + e];
              es[q][e][0] = fma(ys, ys, es[q][e][0]);
              es[q][e][1] = fma(ys, yc, es[q][e][1]);
              es[q][e][2] = fma(yc, yc, es[q][e][2]);
              acc[NMBW - 1][q][e] = acc[NMBW - 1][q][2 + e] = 0.0;
            }
          }
      }
      if ((c + 1) % C::FLUSH == 0 && c + 1 < nch && !FFP_DBG(ar, 4)) {
        // fold the level-1 sums into the level-2 totals of this CTA's scratch slab
#pragma unroll
        for (int r = 0; r < NMBW; ++r)
#pragma unroll
          for (int q = 0; q < NMT; ++q)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              if (ECORR && r == NMBW - 1 && slot_warp) continue;  // open epoch sums stay in registers
              // the slot is private to this thread: first block stores, later blocks add with a
              // fire-and-forget reduction (RED.ADD.F64) -- a load/add/store chain would expose one L2
              // round trip per accumulator
              double* a = sl + (size_t)((r * NMT + q) * 4 + e) * C::NTC;
              if (flushed) atomicAdd(a, acc[r][q][e]);
              else __stcg(a, acc[r][q][e]);
              acc[r][q][e] = 0.0;
            }
        if (ECORR && slot_warp) {
#pragma unroll
          for (int q = 0; q < NMT; ++q)
#pragma unroll
            for (int e = 0; e < 6; ++e) {
              double* a = sl + (size_t)(C::NACC + q * 6 + e) * C::NTC;
              if (flushed) atomicAdd(a, es[q][e / 3][e % 3]);
              else __stcg(a, es[q][e / 3][e % 3]);
              es[q][e / 3][e % 3] = 0.0;
            }
        }
        flushed = true;
      }
    }
    g += (uint32_t)nch;

    // ---- epilogue ------------------------------------------------------------------------
    if (flushed) {
      __threadfence();  // the reductions above are complete before the read-back
#pragma unroll
      for (int r = 0; r < NMBW; ++r)
#pragma unroll
        for (int q = 0; q < NMT; ++q)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (!(ECORR && r == NMBW - 1 && slot_warp)) acc[r][q][e] += __ldcg(sl + (size_t)((r * NMT + q) * 4 + e) * C::NTC);
      if (ECORR && slot_warp) {
#pragma unroll
        for (int q = 0; q < NMT; ++q)
#pragma unroll
          for (int e = 0; e < 6; ++e) es[q][e / 3][e % 3] += __ldcg(sl + (size_t)(C::NACC + q * 6 + e) * C::NTC);
      }
    }
    // this thread holds Y of the tile frequency 8*(wn*NMT + q) + (lane>>2) for the rows 8*(wm*NMBW + r) +
    // 2*(lane&3) + e: acc[r][q][e] is the sin column, acc[r][q][2 + e] the cos column
    // b-sums: one fma chain per row residue j%8 over the warp's row blocks, then a pairwise tree over the 8 residues --
    // (2t, 2t+1) in registers, then the t-lanes -- so a frequency's sums are rounded the same way whatever the MMA
    // shape and the lane that owns a row
    const int mfix = pm.mfix;  // rows below mfix enter the b-sums (plain Fp: mfix = m)
    double* redB = sm.red;  // [WMW][KF][3]
#pragma unroll
    for (int q = 0; q < NMT; ++q) {
      double ps[2][3] = {{0, 0, 0}, {0, 0, 0}};  // (ss, sc, cc) of rows 2t, 2t+1 mod 8
#pragma unroll
      for (int r = 0; r < NMBW; ++r)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = 8 * (wm * NMBW + r) + 2 * (lane & 3) + e;
        const double ys = acc[r][q][e], yc = acc[r][q][2 + e];
        if (j < mfix) {
          ps[e][0] = fma(ys, ys, ps[e][0]);
          ps[e][1] = fma(ys, yc, ps[e][1]);
          ps[e][2] = fma(yc, yc, ps[e][2]);
        } else if (MODE == SweepMode::Nmfp && j < pm.m) {
          // nmfp: rows of the per-draw block go out as z'
          const int64_t f = f0 + 8 * (wn * NMT + q) + (lane >> 2);
          if (f < ar.F) {
            double* z = ar.nm.z(p, f, (ar.F + 31) >> 5, j - mfix + (ar.nm.mvpad - pm.mvar));
            z[0] = ys;
            z[16] = yc;
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (ECORR && slot_warp) {  // the block-N correction enters exactly like the Woodbury b-sums, per slot
          ps[0][k] += es[q][0][k];
          ps[1][k] += es[q][1][k];
        }
        double v = ps[0][k] + ps[1][k];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        if ((lane & 3) == 0) redB[(wm * C::KF + 8 * (wn * NMT + q) + (lane >> 2)) * 3 + k] = v;
      }
    }
    __syncthreads();  // B3: reductions (consumer b-sums, producer scalar sums) published
    const int64_t fidx = f0 + tid;
    if (tid < C::KF && fidx < ar.F) {
      const double* redA = sm.red + C::WMW * C::KF * 3;  // [KSPLIT][KF][5]
      double b[3] = {0, 0, 0}, a[5] = {0, 0, 0, 0, 0};
      for (int w2 = 0; w2 < C::WMW; ++w2)
#pragma unroll
        for (int k = 0; k < 3; ++k) b[k] += redB[(w2 * C::KF + tid) * 3 + k];
      for (int g2 = 0; g2 < C::KSPLIT; ++g2)
#pragma unroll
        for (int k = 0; k < 5; ++k) a[k] += redA[(g2 * C::KF + tid) * 5 + k];
      if (MODE == SweepMode::Fp) {
        if (p < ar.rg.first) ar.fp.put(p, fidx, ar.F, sm.fq[tid], a[0] - b[0], a[1] - b[1], a[2] - b[2], a[3], a[4]);
        else ar.rg.put(p, fidx, ar.F, sm.fq[tid], a, b);
      }
      if (MODE == SweepMode::Nmfp) ar.nm.put_a(p, fidx, (ar.F + 31) >> 5, a[0] - b[0], a[1] - b[1], a[2] - b[2], a[3], a[4]);
      if (MODE == SweepMode::Res) {
        // M of this frequency for every realisation; slot 0 of redB for this frequency is read by this thread only
        redB[tid * 3 + 0] = a[0] - b[0];
        redB[tid * 3 + 1] = a[1] - b[1];
        redB[tid * 3 + 2] = a[2] - b[2];
        ar.res.put_m(p, fidx, sm.fq[tid], a[0] - b[0], a[1] - b[1], a[2] - b[2]);
      }
    }
    if (MODE == SweepMode::Res) res_tail<C>(ar.res, ar.F, sm, acc, redB, p, f0, pm.m, wm, wn, lane);
    __syncthreads();  // B4: fq, red and s_work are reused by the next work item
  }
}

template <class C, SweepMode MODE, bool ECORR>
__global__ void __launch_bounds__(C::NTHREADS, CTAS_PER_SM) fp_sweep_kernel(const SweepArgs ar) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SweepSmem<C> sm(smem_raw);
  __shared__ int s_work;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < C::SST; ++s) { mbar_init(&sm.s_full[s], C::NWP); mbar_init(&sm.s_empty[s], C::NWC); }
    for (int s = 0; s < C::GST; ++s) { mbar_init(&sm.g_full[s], 1); mbar_init(&sm.g_empty[s], C::NWC); }
    for (int s = 0; s < VST; ++s) { mbar_init(&sm.v_full[s], 1); mbar_init(&sm.v_empty[s], C::NWP); }
    fence_barrier_init();
  }
  __syncthreads();
  if (wid < C::NWC) {
    reg_alloc<C::CREGS>();
    consumer_loop<C, MODE, ECORR>(ar, sm, &s_work, wid, lane);
  } else {
    reg_dealloc<C::PREGS>();
    producer_loop<C>(ar, sm, &s_work, wid - C::NWC, lane);
  }
}

// ---- launch helpers -------------------------------------------------------------------------
template <class C, SweepMode MODE, bool ECORR>
int launch_sweep_cfg(const fastfp_pack* pk, const GroupView& g, const SweepArgs& base, cudaStream_t st) {
  static bool attr_done[64] = {};
  if (!attr_done[pk->device & 63]) {
    FFP_CUDA(cudaFuncSetAttribute(fp_sweep_kernel<C, MODE, ECORR>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    attr_done[pk->device & 63] = true;
  }
  SweepArgs a = base;
  a.pidx = g.pidx;
  const int64_t ntile = (a.F + C::KF - 1) / C::KF;
  const int64_t nwork = ntile * g.count;
  if (nwork > 0x7fffffffLL) { set_error("frequency batch too large for one launch"); return -1; }
  a.ntile_f = (int)ntile;
  a.nwork = (int)nwork;
  const int64_t resident = (int64_t)CTAS_PER_SM * pk->num_sms;
  const unsigned grid = (unsigned)(nwork < resident ? nwork : resident);
  FFP_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), st));
  fp_sweep_kernel<C, MODE, ECORR><<<grid, C::NTHREADS, C::SMEM, st>>>(a);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// one translation unit per configuration family instantiates these (compile time)
int dispatch_sweep_w1(const fastfp_pack*, const GroupView&, const SweepArgs&, SweepMode, cudaStream_t);
int dispatch_sweep_w2(const fastfp_pack*, const GroupView&, const SweepArgs&, SweepMode, cudaStream_t);
int dispatch_sweep_w4(const fastfp_pack*, const GroupView&, const SweepArgs&, SweepMode, cudaStream_t);
int dispatch_sweep_wide(const fastfp_pack*, const GroupView&, const SweepArgs&, SweepMode, cudaStream_t);
int dispatch_sweep_xwide(const fastfp_pack*, const GroupView&, const SweepArgs&, SweepMode, cudaStream_t);

// six kernels per configuration: Fp, Nmfp and Res, each with diagonal or block-diagonal N (pk->ecorr; Res: plain-Fp packs
// only, whose residual packets keep the 8 slot rows last, behind the realisations)
#define FFP_SWEEP_CASE(NMBWv, NNBv, WMWv, CIv) \
  FFP_SWEEP_CASE_W(NMBWv, NNBv, WMWv, CIv, NWC, NWP, CONSUMER_REGS, PRODUCER_REGS)
#define FFP_SWEEP_CASE_W(NMBWv, NNBv, WMWv, CIv, NWCv, NWPv, CREGSv, PREGSv)                       \
  if (g.cfg.nmbw == NMBWv && g.cfg.nnb == NNBv && g.cfg.wmw == WMWv && g.cfg.ci == CIv &&          \
      g.cfg.nwc == NWCv) {                                                                         \
    using Cfg_ = SweepCfg<NMBWv, NNBv, WMWv, CIv, NWCv, NWPv, CREGSv, PREGSv>;                      \
    if (mode == SweepMode::Res)                                                                    \
      return pk->ecorr ? launch_sweep_cfg<Cfg_, SweepMode::Res, true>(pk, g, a, st)                \
                       : launch_sweep_cfg<Cfg_, SweepMode::Res, false>(pk, g, a, st);              \
    if (mode == SweepMode::Nmfp)                                                                   \
      return pk->ecorr ? launch_sweep_cfg<Cfg_, SweepMode::Nmfp, true>(pk, g, a, st)               \
                       : launch_sweep_cfg<Cfg_, SweepMode::Nmfp, false>(pk, g, a, st);             \
    return pk->ecorr ? launch_sweep_cfg<Cfg_, SweepMode::Fp, true>(pk, g, a, st)                   \
                     : launch_sweep_cfg<Cfg_, SweepMode::Fp, false>(pk, g, a, st);                 \
  }

}  // namespace ffp
