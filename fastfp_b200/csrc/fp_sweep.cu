// Host side of the sweep: configuration choice, launches, and the ordered pulsar sum.
#include <cstdlib>

#include "fp_sweep_kernel.cuh"

namespace ffp {

// Kernel configuration for a basis of width m (DESIGN.md section 4). A consumer warp owns NMBW
// blocks of 8 basis rows x NNB blocks of 4 frequencies; wider bases put more consumer warps along
// the row direction and fewer frequencies in a tile.
bool sweep_config(int m, KernelCfg* c) {
  if (m < 1 || m > MAX_M) return false;
  if (m <= 40) { *c = {(m + 7) / 8, 4, 1, 16}; return true; }    // 128 frequencies per CTA
  // 64 frequencies per CTA on 8 consumer + 8 producer warps (fp_sweep_w2.cu): a producer warp owns a group of 8
  // frequencies and evaluates its sincos chains four at a time, and the 512-thread register pool leaves the consumers
  // spill-free. (8 producer warps at one chain each fall behind the MMAs: a 12-consumer/8-producer split measured
  // -6% net for m = 72.)
  if (m <= 80) { *c = {(m + 7) / 8, 2, 1, 32}; return true; }
  if (m <= 160) { *c = {(m + 15) / 16, 2, 2, 16}; return true; }  // 32 frequencies per CTA
  if (m <= 320) { *c = {(m + 31) / 32, 2, 4, 16}; return true; }  // 16 frequencies per CTA
  // all eight consumer warps along the rows, chunks of 8 TOAs (the G tile of a chunk is 8 x 640 doubles = 40 KB): 8
  // frequencies per CTA. Real pulsars with many DMX columns land here; the tile is reused across 8 frequencies only, so
  // this family runs at a lower fraction of the pipe than the narrow ones (SURVEY.md section 7.3-H3).
  *c = {(m + 63) / 64, 2, 8, 8};                                  // m <= 640
  return true;
}

// NACC <= 80, at most 12 consumer warps; producers keep 5 * SPW * XW <= 10 slots per thread, 512 threads at most
int sweep_max_slab_doubles() { return (40 + 12) * 12 * 32 + 10 * NTP; }

static int dispatch_group(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode,
                          cudaStream_t st) {
  if (g.cfg.wmw == 8) return dispatch_sweep_xwide(pk, g, a, mode, st);
  if (g.cfg.wmw == 4) return dispatch_sweep_wide(pk, g, a, mode, st);
  if (g.cfg.wmw == 1 && g.cfg.nnb == 4) return dispatch_sweep_w1(pk, g, a, mode, st);
  if (g.cfg.wmw == 1) return dispatch_sweep_w2(pk, g, a, mode, st);
  return dispatch_sweep_w4(pk, g, a, mode, st);
}

static SweepArgs sweep_args(const double* packets, const PulsarMeta* meta, const fastfp_pack* pk,
                            const double* d_freqs, int64_t F) {
  SweepArgs a{};
  a.packets = packets;
  a.meta = meta;
  a.freqs = d_freqs;
  a.F = F;
  a.slab = pk->core.slab.get();
  a.counter = pk->core.counter.get();
  return a;
}

// the pack's sweep in mode Fp or Nmfp; rest_only: only the pulsars the tensor sweep left out
static int launch_fp_groups(const fastfp_pack* pk, SweepArgs a, SweepMode mode, bool rest_only, cudaStream_t st) {
#ifdef FFP_DEBUG_SWITCHES  // profiling builds only; the shipped library is compiled without it
  static const int dbg = getenv("FASTFP_DBG") ? atoi(getenv("FASTFP_DBG")) : 0;
  a.dbg = dbg;
#endif
  a.done_mask = pk->core.done_mask.get();
  for (const Group& g : pk->groups) {
    const GroupView v = rest_only ? g.rest() : g.all();
    if (v.count == 0) continue;
    if (int rc = dispatch_group(pk, v, a, mode, st)) return rc;
  }
  return 0;
}

// Row groups (DESIGN.md section 5h): per (wide pulsar, frequency), M = ((sNs - b_0) - b_1) - ... in group order for
// ss, sc and cc, then the term and the inner products exactly as FpOut::put writes those of a whole pulsar
__global__ void row_group_combine_kernel(const int* __restrict__ wide, const double* __restrict__ freqs, int64_t F,
                                         const FpOut out, const RowGroupOut rg) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int* wl = wide + RG_WIDE * blockIdx.y;
  const int p = wl[0], k1 = wl[2] - rg.first - rg.nwide, g = wl[3];
  const double* a = rg.part_at(blockIdx.y, f, F);
  double ss = a[0], sc = a[1], cc = a[2];
  for (int k = 1; k < g; ++k) {
    const double* b = rg.b_at(k1 + k - 1, f, F);
    ss -= b[0];
    sc -= b[1];
    cc -= b[2];
  }
  const double fq = freqs[f];
  out.put(p, f, F, fq, ss, sc, cc, a[3], a[4]);
}

int launch_fp_sweep(const fastfp_pack* pk, const double* d_freqs, int64_t F, const FpOut& out, cudaStream_t st,
                    bool rest_only) {
  SweepArgs a = sweep_args(pk->core.packets.get(), pk->core.meta.get(), pk, d_freqs, F);
  a.fp = out;
  a.rg = RowGroupOut{nullptr, nullptr, pk->P, pk->n_wide};  // meta indices >= P are row-group items
  if (pk->n_wide) {
    if (int rc = pk->rg.grow(pk->rg_doubles_per_freq() * F)) return rc;
    a.rg.part = pk->rg.get();
    a.rg.b = pk->rg.get() + 5 * (int64_t)pk->n_wide * F;
  }
  if (int rc = launch_fp_groups(pk, a, SweepMode::Fp, rest_only, st)) return rc;
  if (!pk->n_wide) return 0;
  row_group_combine_kernel<<<dim3((unsigned)((F + 255) / 256), (unsigned)pk->n_wide), 256, 0, st>>>(
      pk->core.wide.get(), d_freqs, F, out, a.rg);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

int launch_fp_sweep(const fastfp_pack* pk, const double* d_freqs, int64_t F, const NmfpTiles& out, cudaStream_t st,
                    bool rest_only) {
  SweepArgs a = sweep_args(pk->core.packets.get(), pk->core.meta.get(), pk, d_freqs, F);
  a.nm = out;
  return launch_fp_groups(pk, a, SweepMode::Nmfp, rest_only, st);
}

// The residual batch (DESIGN.md sections 5d, 5e): the fp64 kernel on the pack's residual packets, whose G tiles carry
// the realisations' w_k as extra rows
int launch_fp_sweep_res(const fastfp_pack* pk, const double* d_freqs, int64_t F, const ResOut& out, cudaStream_t st) {
  SweepArgs a = sweep_args(pk->res.packets.get(), pk->res.meta.get(), pk, d_freqs, F);
  a.res = out;
  a.done_mask = pk->res.done_mask.get();  // block-N packs: the slot masks of the residual layout's chunks
  for (const Group& g : pk->res.groups)
    if (int rc = dispatch_group(pk, g.all(), a, SweepMode::Res, st)) return rc;
  return 0;
}

// out[k * ld + f] = sum over pulsars of terms[k][p][f], in pulsar order from 0 (fastfp.py:71,90)
__global__ void reduce_terms_rows_kernel(const double* __restrict__ terms, int P, int64_t F,
                                         double* __restrict__ out, int64_t ld) {
  const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const double* t = terms + (size_t)blockIdx.y * P * F;
  double acc = 0.0;
  for (int p = 0; p < P; ++p) acc += t[(size_t)p * F + f];
  out[(size_t)blockIdx.y * ld + f] = acc;
}

int launch_reduce_terms_rows(const double* d_terms, int R, int P, int64_t F, double* d_out, int64_t ld,
                             cudaStream_t st) {
  reduce_terms_rows_kernel<<<dim3((unsigned)((F + 255) / 256), (unsigned)R), 256, 0, st>>>(d_terms, P, F, d_out, ld);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ffp
