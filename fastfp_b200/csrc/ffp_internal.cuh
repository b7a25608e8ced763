// Internal declarations shared by the CUDA translation units of libfastfp_b200.so.
// sm_90a only (built with -gencode arch=compute_90a,code=sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/fastfp_b200.h"

namespace ffp {

// ---- tiling constants of the sweep kernel (DESIGN.md section 4) -------------------------
constexpr int NWC = 8;         // consumer (MMA) warps per sweep CTA: two per SM sub-partition
constexpr int NWP = 16;        // producer (sincos) warps per sweep CTA by default: four per SM sub-partition
constexpr int NTC = NWC * 32, NTP = NWP * 32;
constexpr int CTAS_PER_SM = 1;
constexpr int CONSUMER_REGS = 120, PRODUCER_REGS = 56;  // default setmaxnreg split of the 768 x 80 pool
constexpr int VST = 16;        // TOA-vector ring depth (t | 1/N | w; TMA -> producer)
constexpr int FLUSH_TOAS = 512;  // level-1 accumulation block, in TOAs
constexpr int MAX_M = 640;     // widest basis the sweep kernel handles (8 warp rows x 10 blocks of 8 rows)
// Wider bases (diagonal-N Fp packs only, DESIGN.md section 5h) are swept as row groups of G, each one work item of the
// kernel: ceil(m / RG_ROWS) groups of near-equal width in whole blocks of 8 rows, up to MAX_M_WIDE columns. Groups of at
// most 288 rows run on the 16-frequency family with at most 9 row blocks per warp, measured at 0.57-0.59 ns per
// (frequency, pulsar, G row) on an H100, against 1.06 at 10 blocks (320 rows) and 0.90-0.94 on the 8-frequency family
// (DESIGN.md section 5h)
constexpr int RG_ROWS = 288;
constexpr int MAX_M_WIDE = 2688;  // 10 groups of 264-272 rows
constexpr int MAX_RG = (MAX_M_WIDE + RG_ROWS - 1) / RG_ROWS;

// the row groups of a basis of width m (1: the whole basis is one work item) and the first row of group k (k == groups:
// m); the one statement of the split rule
__host__ __device__ inline int row_groups(int m) { return m <= MAX_M ? 1 : (m + RG_ROWS - 1) / RG_ROWS; }
__host__ __device__ inline int row_group_start(int m, int k) {
  const int nb = (m + 7) / 8, g = row_groups(m);
  const int r = 8 * (k * (nb / g) + (k < nb % g ? k : nb % g));
  return r < m ? r : m;
}

// G rows a pulsar of basis width m takes in the sweep kernel: its basis rows, then R residual realisations from row
// roundup8(m) on (residual batches, DESIGN.md section 5d), then with a block-diagonal N the 8 epoch-slot rows last
inline int sweep_rows(int m, int64_t R, bool blockn) {
  return (m + 7) / 8 * 8 + (int)((R + 7) / 8 * 8) + (blockn ? 8 : 0);
}

// Sweep configuration. The contraction runs on the fp64 MMA path (mma.sync.m16n8k4.f64, basis rows on the N side): a
// warp owns NMBW row blocks (8 basis rows each) x NNB/2 tiles of 8 frequencies x {sin, cos} (the 16 MMA rows), i.e.
// 4*NNB frequencies; WMW consumer warps split the rows, NWC/WMW split the frequencies of the tile.
//   CI  TOAs per staged chunk (KB = CI/4 k-blocks)
//   NWC / NWP  consumer (MMA) / producer (sincos) warps of the CTA. The default is two consumer and four
//   producer warps per SM sub-partition (8 + 16), where a producer evaluates one sincos chain at a time; the
//   m <= 80 family runs 8 + 8, whose producers have the registers to evaluate four chains in lockstep.
//   CREGS / PREGS  setmaxnreg split of the launch-time register pool (NTHREADS x the launch register count)
template <int NMBW_, int NNB_, int WMW_, int CI_, int NWC_ = ffp::NWC, int NWP_ = ffp::NWP,
          int CREGS_ = CONSUMER_REGS, int PREGS_ = PRODUCER_REGS>
struct SweepCfg {
  static constexpr int NMBW = NMBW_, NNB = NNB_, WMW = WMW_, CI = CI_;
  static constexpr int NWC = NWC_, NWP = NWP_, NTC = NWC_ * 32, NTP = NWP_ * 32, NTHREADS = NTC + NTP;
  static constexpr int CREGS = CREGS_, PREGS = PREGS_;
  static_assert(NTHREADS <= 1024 && NWC % WMW_ == 0, "warp layout");
  static_assert(NTC * CREGS + NTP * PREGS <= NTHREADS * ((65536 / NTHREADS) / 8 * 8), "register pool");
  static constexpr int WNW = NWC / WMW;        // consumer warps along frequency
  static constexpr int KF = WNW * NNB * 4;     // frequencies per CTA
  static constexpr int NMB = NMBW * WMW;       // row blocks
  static constexpr int MP = 8 * NMB;           // padded basis width (rows of G)
  static constexpr int KB = CI / 4;            // k-blocks (4 TOAs) per chunk
  static constexpr int ST = CI * 2 * KF;       // doubles of one sin/cos tile: [KB][NX][32][2]
  static constexpr int VEC = 4 * CI;           // doubles of the vector part: (t, 1/N, w, 0) per TOA
  static constexpr int GT = CI * MP;           // doubles of the G part: [KB][NMB][32] fragments
  static constexpr int PK = VEC + GT;          // doubles per packet
  // basis phase: one warp store covers 8 frequencies x 4 TOAs; a thread keeps XW frequencies
  static constexpr int NX = KF / 8;                       // groups of 8 frequencies
  static constexpr int XW = NX >= NWP ? NX / NWP : 1;      // frequency groups per producer warp
  // the five scalar sums of a group are kept as KSPLIT partial sums over consecutive k-block ranges, added in order
  // in the epilogue. The partition is the one the default 16 producer warps give (warps sharing a group split its
  // k-blocks), whatever NWP is, so a frequency's sums are rounded the same way under every producer split.
  static constexpr int KSPLIT = NX >= ffp::NWP ? 1 : (ffp::NWP / NX < KB ? ffp::NWP / NX : KB);
  static constexpr int KBW = KB / KSPLIT;                 // k-blocks of one partial sum
  // producer warps sharing one group, and the partial sums each of them keeps; with few groups and few k-blocks
  // the surplus warps stay idle (they still take part in the barrier protocol)
  static constexpr int WPG = NX >= NWP ? 1 : (NWP / NX < KSPLIT ? NWP / NX : KSPLIT);
  static constexpr int SPW = KSPLIT / WPG;
  static constexpr int NACTIVE = NX >= NWP ? NWP : NX * WPG;  // producer warps with work
  // sincos chains a producer thread evaluates in lockstep (sincos_cw_n): lockstep chains need about 72 registers,
  // so with fewer a thread evaluates one (TOA, frequency) pair at a time
  static constexpr int NV = PREGS >= 72 ? KBW * XW : 1;
  static constexpr int NACC = 2 * NMBW * NNB;  // accumulators per thread
  static constexpr int NACCX = NACC + 3 * NNB;  // + epoch sums of the block-N variant
  static constexpr int SLAB = NACCX * NTC + 5 * SPW * XW * NTP;  // doubles of level-2 scratch per CTA
  static constexpr int FLUSH = FLUSH_TOAS / CI;  // chunks per level-1 block
  // ring depths: sin/cos tiles (producer -> consumer) and G tiles (TMA -> consumer), as deep as
  // the shared-memory budget allows
  static constexpr int SST = ST * 8 * 8 <= 140 * 1024 ? 8 : 4;
  static constexpr int GBUDGET = 214 * 1024 - SST * ST * 8 - VST * VEC * 8;
  static constexpr int GST = GBUDGET / (GT * 8) >= 8 ? 8 : (GBUDGET / (GT * 8) >= 2 ? GBUDGET / (GT * 8) : 2);
  static constexpr int RED = KF * (3 * WMW + 5 * KSPLIT);  // doubles of epilogue reduction scratch
  static constexpr size_t SMEM =
      (size_t)(SST * ST + GST * GT + VST * VEC + KF + RED + 2 * (SST + GST + VST)) * 8 + 128;
  static_assert(KB % KSPLIT == 0 && KSPLIT % WPG == 0 && NACTIVE <= NWP && (KBW * XW) % NV == 0,
                "basis-phase mapping");
  static_assert(GST >= 3, "the consumers prefetch across chunk boundaries: three G stages at least");
};

// offset of G element (TOA il within its chunk, basis row j) inside a packet's G part:
// fragment order [k-block][row block][lane], lane = (j%8)*4 + il%4 -- the B-operand layout of
// mma.m16n8k4 (n = lane>>2, k = lane&3), so a warp's fragment load is 256 contiguous bytes.
__host__ __device__ inline int g_frag_index(int il, int j, int nmb) {
  return (((il >> 2) * nmb + (j >> 3)) << 5) + (((j & 7) << 2) | (il & 3));
}

// Per-pulsar descriptor, device-visible.
struct PulsarMeta {
  int64_t pk_off;  // offset (in doubles) of the pulsar's first packet inside `packets`
  int64_t L_off;   // offset of its m x m factor inside `Lbuf`
  int64_t raw_off; // offset of its TOA-length vectors inside the staging arrays
  int64_t T_off;   // offset of its raw T inside the staging array
  int32_t n, m, nch, mpad;
  int32_t mfix, mvar;  // nmfp: leading draw-independent columns / trailing per-draw columns
  int32_t var_off;     // nmfp: offset of this pulsar's varying block in a phiinv_var row
  int32_t ci;          // TOAs per packet for this pulsar's kernel configuration
  double tabs_max;     // max |TOA| (inf if any TOA is not finite): decides the sincos path per tile
  int64_t dm_off;      // block-N packs: offset of this pulsar's per-chunk slot masks
  int64_t i8_off;      // tensor path: byte offset of this pulsar's digit-plane stages
  int32_t i8_rows;     // tensor path: rows stored per plane (basis rows + the w row, padded to 8)
  int32_t i8_nst;      // tensor path: stages of 32 TOAs
  double ninv_sum;     // tensor path: sum_i 1/N_i (c N^-1 c = sum 1/N - s N^-1 s, so the producers form two sums, not three)
};
// Row groups (DESIGN.md section 5h): the device meta holds the P pulsars, then one work item per row group of each wide
// pulsar, each with the pulsar's entry except its own ci, nch, mpad, pk_off and m = mfix = its row count -- first group 0
// of every wide pulsar, in pulsar order, then the other groups, pulsar by pulsar in group order. A wide pulsar's own
// entry describes the whole basis and is not swept. PackCore::wide lists per wide pulsar RG_WIDE ints: the pulsar, the
// meta index of its group 0, that of its group 1 (groups 2 ... follow it) and its number of groups.
constexpr int RG_WIDE = 4;

struct KernelCfg {  // run-time mirror of SweepCfg's parameters
  int nmbw, nnb, wmw, ci;
  int nwc = NWC;  // consumer warps (8, or 12 for the three-row-group configurations)
  int kf() const { return (nwc / wmw) * nnb * 4; }
  int mp() const { return 8 * nmbw * wmw; }
  bool operator<(const KernelCfg& o) const {
    if (nmbw != o.nmbw) return nmbw < o.nmbw;
    if (nnb != o.nnb) return nnb < o.nnb;
    if (wmw != o.wmw) return wmw < o.wmw;
    if (nwc != o.nwc) return nwc < o.nwc;
    return ci < o.ci;
  }
};

extern std::atomic<int64_t> g_launches;
extern std::atomic<int64_t> g_device_bytes;  // device memory this library holds (fastfp_device_bytes)
void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);

#define FFP_CUDA(call)                                         \
  do {                                                         \
    cudaError_t e__ = (call);                                  \
    if (e__ != cudaSuccess) return ffp::cuda_fail(e__, #call); \
  } while (0)

// ---- owners: every allocation of the library is released by its holder, on every path -----------
// device memory: allocated only by dev_alloc, which counts it in g_device_bytes; the deleter takes the count back
struct CudaFree {
  size_t bytes = 0;
  void operator()(void* p) const {
    cudaFree(p);
    g_device_bytes -= (int64_t)bytes;
  }
};
template <typename T>
using DeviceBuf = std::unique_ptr<T, CudaFree>;
// count elements of T into *buf; the buffer it held before is released after the new allocation (Scratch::grow
// releases first where the two must not coexist)
template <typename T>
inline cudaError_t dev_alloc(DeviceBuf<T>* buf, size_t count) {
  T* p = nullptr;
  const size_t bytes = count * sizeof(T);
  const cudaError_t e = cudaMalloc(&p, bytes);
  if (e != cudaSuccess) {
    buf->reset();
    return e;
  }
  g_device_bytes += (int64_t)bytes;
  *buf = DeviceBuf<T>(p, CudaFree{bytes});
  return e;
}
// pinned host memory
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <typename T>
using PinnedBuf = std::unique_ptr<T, CudaFreeHost>;
template <typename T>
inline cudaError_t pinned_alloc(PinnedBuf<T>* buf, size_t count) {
  T* p = nullptr;
  const cudaError_t e = cudaMallocHost(&p, count * sizeof(T));
  buf->reset(e == cudaSuccess ? p : nullptr);
  return e;
}
// events
struct CudaEventDestroy {
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, CudaEventDestroy>;
inline cudaError_t event_create(Event* ev, unsigned flags = cudaEventDefault) {
  cudaEvent_t e = nullptr;
  const cudaError_t rc = cudaEventCreateWithFlags(&e, flags);
  ev->reset(rc == cudaSuccess ? e : nullptr);
  return rc;
}

// the pulsars one sweep launch takes: a configuration and a device list of pulsar indices
struct GroupView {
  KernelCfg cfg;
  const int* pidx;
  int count;
};
struct Group {  // pulsars that share one kernel instantiation
  KernelCfg cfg;
  int count = 0;
  DeviceBuf<int> pidx;       // their indices
  int count_rest = 0;        // ... those of them the tensor sweep does not take (build_i8_planes), when it takes some
  DeviceBuf<int> pidx_rest;
  GroupView all() const { return {cfg, pidx.get(), count}; }
  GroupView rest() const { return {cfg, pidx_rest.get(), count_rest}; }
};

// device memory a pack keeps for its calls: grown on demand (contents are not preserved), kept until released
template <typename T>
struct Scratch {
  DeviceBuf<T> buf;
  int64_t cap = 0;
  T* get() const { return buf.get(); }
  int grow(int64_t need) {
    if (cap >= need) return 0;
    release();  // before the new allocation: the old and the new buffer are never held together
    FFP_CUDA(dev_alloc(&buf, (size_t)need));
    cap = need;
    return 0;
  }
  void release() {
    buf.reset();
    cap = 0;
  }
};

// ---- the memory of a pack, one owner per feature that creates it ----------------------------------
// Releasing a feature replaces its struct with an empty one.

// every pack (pack_layout; the slot masks: block-N packs, stage_slots)
struct PackCore {
  DeviceBuf<PulsarMeta> meta;          // [P + row-group items]
  DeviceBuf<int> wide;                 // [RG_WIDE x wide pulsars] (row groups, see PulsarMeta)
  DeviceBuf<double> packets;           // [sum_p nch_p][PK_p]
  DeviceBuf<double> L;                 // Cholesky factors (Fp) / fixed-block factors (nmfp)
  DeviceBuf<int> info;                 // per-pulsar factorisation status
  DeviceBuf<double> slab;              // level-2 accumulation scratch, one slab per resident CTA
  DeviceBuf<unsigned int> counter;     // persistent-CTA work counter
  DeviceBuf<unsigned char> done_mask;  // block-N: per-chunk epoch-slot masks
};

// INT8 tensor-core path (fp_sweep_i8.cu, build_i8_planes): digit planes of G, per-row scales
struct TensorPath {
  DeviceBuf<unsigned char> planes;
  DeviceBuf<double> scale;  // [P][128]
  DeviceBuf<int> pidx;      // pulsars on the tensor sweep (all of them, or those that fit: n <= 16384, finite planes)
  int count = 0;            // their number; the others stay on the fp64 kernel in the same sweep
  bool ok = false;          // the planes exist
  int rows_max = 0;
};

// nmfp packs (nmfp_pack_finish)
struct NmfpState {
  DeviceBuf<double> S0;  // [P][mvpad][mvpad] Schur complement of the fixed block (no phiinv)
  DeviceBuf<double> zr;  // [P][mvpad]  z'_r
};

// staging of the per-draw power-law parameters (fastfp_powerlaw_phiinv): device + pinned host copy of cap doubles;
// the event marks the last H2D copy out of the host copy; tab is the frequency table already on the device
struct PowerlawStaging {
  DeviceBuf<double> dev;
  PinnedBuf<double> host;
  Event event;
  int64_t cap = 0;
  std::vector<double> tab;
};

// residual batch (fastfp_pack_set_residuals, DESIGN.md section 5d): per pulsar, the G rows followed by the R
// realisations' w_k rows, in packets of the kernel configuration for its sweep_rows (block-N packs,
// fastfp_pack_set_residuals_blockn: with the epoch slots last; their TOAs in the layout of that configuration's chunk
// size, with its own slot masks)
struct ResidualBatch {
  DeviceBuf<double> packets;
  DeviceBuf<PulsarMeta> meta;
  DeviceBuf<unsigned char> done_mask;  // block-N: per-chunk epoch-slot masks of the residual layout
  std::vector<Group> groups;
  mutable Scratch<double> terms;  // [R][P][F_batch] terms of one frequency batch
  int64_t R = 0;
  int64_t bytes = 0;
};

}  // namespace ffp

// The opaque handle of include/fastfp_b200.h.
struct fastfp_pack {
  int device = 0;
  int P = 0;
  int num_sms = 0;
  bool nmfp = false;
  bool ecorr = false;            // block-diagonal N (kernel ECORR): 8 epoch-slot rows in the G tiles
  std::vector<ffp::PulsarMeta> meta;
  std::vector<ffp::PulsarMeta> items;  // the row-group work items, meta indices P ... (DESIGN.md section 5h)
  int n_wide = 0;                       // pulsars with row groups
  std::vector<ffp::Group> groups;
  std::vector<int> info;         // host copy of core.info, read back when the pack is built (fastfp_pack_factor_info)
  ffp::PackCore core;
  ffp::TensorPath i8;            // chosen per pack (path)
  int path = 0;                  // FASTFP_PATH_AUTO / _FP64 / _I8 / _MIXED (fastfp_pack_set_path)
  // AUTO resolves to the fp64 DMMA kernel: on an H100 it sweeps m = 72 bases about twice as fast as the tensor kernel
  // (C2: 35 ms against 78 ms per step, 400 W H100 SXM). I8 and MIXED select the tensor kernel.
  bool use_i8() const { return i8.ok && (path == FASTFP_PATH_I8 || path == FASTFP_PATH_MIXED); }
  bool i8_all() const { return i8.count == P; }
  int64_t bytes = 0;
  int64_t mvar_total = 0;
  int mvar_max = 0;
  int mvpad = 0;           // nmfp: per-draw block width padded to the stage-B tile (32, 64 or 96)
  ffp::NmfpState nm;
  // scratch reused across sweeps
  mutable ffp::Scratch<double> terms;
  mutable ffp::Scratch<double> freqs;
  mutable ffp::Scratch<double> out;
  mutable ffp::Scratch<double> scratch;  // nmfp: stage-A tiles of a frequency batch
  mutable ffp::Scratch<double> lf;       // nmfp: L^-1 fragments of a draw batch
  mutable ffp::Scratch<double> inner;    // Fe-statistic: inner products of a frequency batch + antenna patterns
  mutable ffp::Scratch<double> rg;       // row groups: the partial sums of a frequency batch (RowGroupOut)
  // doubles of row-group scratch per frequency of a sweep (0 without wide pulsars): callers size their batches with it
  int64_t rg_doubles_per_freq() const { return 5 * (int64_t)n_wide + 3 * ((int64_t)items.size() - n_wide); }
  mutable ffp::PowerlawStaging pl;
  ffp::ResidualBatch res;
  // optional per-stage timing of nmfp sweeps (fastfp_nmfp_stage_timing): stage A, factor, stage B
  mutable bool time_stages = false;
  mutable double stage_ms[3] = {0.0, 0.0, 0.0};
};

namespace ffp {

// ---- kernel launchers (defined in the .cu files) ---------------------------------------
// precompute.cu
struct BlockNDev {         // device copies of the block-N (kernel ECORR) side arrays, or all null
  const double* res_w;     // (N^-1 r) * Nvec per TOA
  const int* slot_idx;     // epoch slot (0..7) of a TOA inside its chunk, -1 if none
  const double* slot_val;  // sqrt(beta_e) / Nvec_i
};
int launch_fp_precompute(fastfp_pack* pk, const double* d_toas, const double* d_res,
                         const double* d_Nvec, const double* d_T, cudaStream_t st,
                         double* d_ur_keep = nullptr,  // [P][MAX_M], receives G r
                         const BlockNDev* bn = nullptr);
// host arrays of a residual batch: per pulsar, the residual layout's TOA count n[p] and the (R, n[p]) realisations raw
// and as (N^-1 r_k) * Nvec (diagonal N: the pack's n, and res_w == res); block-N packs also that layout's slot indices
// and values (per TOA) and masks (per chunk), null otherwise
struct ResHost {
  const int64_t* n;
  const double* const* res;
  const double* const* res_w;
  const int32_t* const* slot_idx;
  const double* const* slot_val;
  const unsigned char* const* done_mask;
};
// a residual batch drawn on the device (sim.cu, DESIGN.md section 5g): the stream's seed and first realisation index,
// per pulsar the prior phiinv (m_p), the signal (sig_freq (R), sig_amp (R, P, 2); both null: none); block-N packs also
// per position of the residual layout the original TOA index and the epoch (-1: none), per epoch sqrt(j_e) and beta_e
struct SimHost {
  int64_t seed, first;
  bool noise;
  const double* const* phiinv;
  const double* sig_freq;
  const double* sig_amp;
  const int32_t* const* toa_index;
  const int32_t* const* epoch;
  const double* const* sqrt_j;
  const double* const* beta;
};
// its device side
struct SimArgs {
  uint64_t seed, first;
  int noise;
  const double* sig_freq;  // (R) or null: no signal
  const double* sig_amp;   // (R, P, 2): (A_s, A_c)
  const double* phiinv;    // [P][MAX_M]
  // block-diagonal N (all null for a diagonal N): per position of the (R, n_shared) staging at smeta.raw_off the
  // original TOA index (-1 on padding); the segments, nseg_p + 1 starts per pulsar from seg_off[p] (an epoch's run of
  // positions, or one position outside any epoch), and each one's epoch; per epoch sqrt(j_e) and beta_e from ep_off[p]
  const int* toa_index;
  const int* seg;
  const int* seg_epoch;
  const int64_t* seg_off;
  const double* sqrt_j;
  const double* beta;
  const int64_t* ep_off;
};
// the device arrays of SimArgs and the host arrays their copies read, held until the batch is built
struct SimStage {
  SimArgs args{};
  DeviceBuf<double> phiinv, sig_freq, sig_amp, sqrt_j, beta;
  DeviceBuf<int> toa_index, seg, seg_epoch;
  DeviceBuf<int64_t> seg_off, ep_off;
  std::vector<double> host_phi, host_sqrt_j, host_beta;
  std::vector<int> host_idx, host_seg, host_seg_ep;
  std::vector<int64_t> host_seg_off, host_ep_off;
};
// sim_noise_kernel: the realisations n_k into the (R, n_shared) staging (and res_w for a block N)
int launch_sim_noise(const SimHost& s, const fastfp_pack* pk, const std::vector<PulsarMeta>& smeta,
                     const PulsarMeta* d_smeta, int64_t R, double* d_res, double* d_res_w, SimStage* ss,
                     cudaStream_t st);
// sim_basis_kernel: U[p][k] -= L^-1 (sqrt(phiinv) o zeta), U as ur_batch_kernel writes it (row stride ld)
int launch_sim_basis(const fastfp_pack* pk, int64_t R, double* d_U, int ld, const SimStage& ss, cudaStream_t st);
// the residual packets of R realisations into pk->res, which the caller has released: uploaded from h.res / h.res_w, or
// drawn on the device when sim is set (h then gives the layout only)
int build_res_packets(fastfp_pack* pk, int64_t R, const ResHost& h, cudaStream_t st, const SimHost* sim = nullptr);
// packets of pulsars one after another, each in the kernel configuration for its number of G rows
struct PacketLayout {
  int64_t size = 0;                              // doubles
  std::map<KernelCfg, std::vector<int>> groups;  // the pulsars of each configuration
  // pulsar p with `rows` G rows and pm->n TOAs: sets pm's ci, nch, mpad and pk_off; false if no configuration has them
  bool place(int p, int rows, PulsarMeta* pm);
  // the groups with their indices on the device, appended to *out
  int upload(std::vector<Group>* out) const;
};
// fe.cu
int launch_fe_combine(const double* d_inner, int P, int64_t F, const double* d_fplus, const double* d_fcross, int64_t S,
                      double* d_out, int64_t out_ld, cudaStream_t st);
// sky maximum: d_w = (S, P, 5) weights from launch_fe_sky_weights; a plan with nchunk > 1 needs the (nchunk, F)
// scratch d_part_v / d_part_i for the per-chunk bests
struct FeSkyPlan {
  int64_t chunk;   // sky positions per chunk (a multiple of the pass width)
  int64_t nchunk;  // chunks along the sky axis
};
FeSkyPlan fe_skymax_plan(int64_t F, int64_t S, int num_sms);
int launch_fe_sky_weights(const double* d_fplus, const double* d_fcross, int64_t n, double* d_w, cudaStream_t st);
int launch_fe_skymax(const double* d_inner, int P, int64_t F, const double* d_w, int64_t S, const FeSkyPlan& pl,
                     double* d_part_v, int64_t* d_part_i, double* d_best, int64_t* d_idx, cudaStream_t st);
// sky maximum of a residual batch (DESIGN.md section 5e): d_x = (s|r_k), (c|r_k) as [F][P][R][2] and d_mi = (s|s),
// (s|c), (c|c) as [F][P][3] from launch_fp_sweep_res; d_fplus / d_fcross (S, P). Writes (R, F) with row stride ld; a
// plan with nchunk > 1 needs ld == F and the (nchunk, R, F) scratch d_part_v / d_part_i.
FeSkyPlan fe_skymax_res_plan(int64_t F, int64_t R, int64_t S, int num_sms, bool may_split);
int launch_fe_skymax_res(const double* d_x, const double* d_mi, int P, int64_t R, int64_t F, const double* d_fplus,
                         const double* d_fcross, int64_t S, const FeSkyPlan& pl, double* d_part_v, int64_t* d_part_i,
                         double* d_best, int64_t* d_idx, int64_t ld, cudaStream_t st);
bool sweep_config(int m, KernelCfg* cfg);
int sweep_max_slab_doubles();
// xcy.cu
int launch_tnt(int64_t n, int64_t m, const double* dN, const double* dT, const double* d_phiinv, double* d_part,
               int nsplit, double* d_out, cudaStream_t st);
int launch_xcy(int64_t n, int64_t m, const double* dN, const double* dT, const double* dS,
               const double* dx, const double* dy, const double* dx0, double* d_work, double* d_out,
               cudaStream_t st);  // dx0: raw x for the x^T N^-1 y term (null: dx)
// microbench.cu
int run_fp64_peak(int kind, int iters, double* tflops, double* ms);

// ---- small PTX helpers: mbarrier + 1-D TMA bulk copy ------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      " selp.b32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  while (!mbar_try_wait(bar, parity)) __nanosleep(64);  // back off: polling shares the MIO queue with LDS
}
// for the warps on the critical path (the MMA consumers): try_wait already suspends the warp for a
// hardware-chosen interval and wakes it when the phase completes, so no extra sleep that could overshoot
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- warp-specialised kernels: moving registers between warp roles -------------------------
template <int R>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}

// ---- fp64 MMA -------------------------------------------------------------------------------
// D(8x8) += A(8x4) . B(4x8). Lane l holds A[l>>2][l&3], B[l&3][l>>2], D[l>>2][2*(l&3)+{0,1}].
__device__ __forceinline__ void dmma_m8n8k4(double& d0, double& d1, double a, double b) {
  asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
      : "+d"(d0), "+d"(d1)
      : "d"(a), "d"(b));
}
// D(16x8) += A(16x4) . B(4x8). With g = l>>2, t = l&3, lane l holds A[g][t], A[g+8][t] (a0, a1), B[t][g] (b),
// D[g][2t+{0,1}] (d0, d1) and D[g+8][2t+{0,1}] (d2, d3).
__device__ __forceinline__ void dmma_m16n8k4(double (&d)[4], double a0, double a1, double b) {
  asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a0), "d"(a1), "d"(b));
}

// the quiet NaN the statistics return where they are undefined (f <= 0, an empty sky maximum)
__device__ __forceinline__ double kNaN() { return __longlong_as_double(0x7ff8000000000000LL); }

// One pulsar's term 0.5 N^T M^-1 N with M = [[m00, m01], [m01, m11]], N = [n0, n1], by LU with partial pivoting like
// jnp.linalg.solve (fastfp.py:90, nmfp.py:117). Where M is singular to the last bit (the Earth-term basis lies inside
// span(T), e.g. at f = 1/yr against fitted yearly sinusoids) a pivot is exactly zero; the unknown it would divide out is
// set to zero (the basic solution) so the term stays finite instead of 0/0. NaN inputs still give NaN.
__device__ __forceinline__ double term_2x2(double m00, double m01, double m11, double n0, double n1) {
  const double N0 = n0, N1 = n1;
  double m10 = m01;
  if (fabs(m10) > fabs(m00)) {  // row swap; the unknowns keep their order
    double t0 = m00; m00 = m10; m10 = t0;
    t0 = m01; m01 = m11; m11 = t0;
    t0 = n0; n0 = n1; n1 = t0;
  }
  const double lq = m00 != 0.0 ? m10 / m00 : 0.0;
  const double u = m11 - lq * m01;
  const double x1 = u != 0.0 ? (n1 - lq * n0) / u : 0.0;
  const double x0 = m00 != 0.0 ? (n0 - m01 * x1) / m00 : 0.0;
  return 0.5 * (N0 * x0 + N1 * x1);
}

// ---- the sweep's outputs, one block per mode (DESIGN.md sections 4, 5, 5d, 5e) --------------
// Both sweep kernels write through these. The caller passes the sizes of the launch -- F frequencies, the row length of
// every output, and nt32 = ceil(F / 32) -- and the frequency value fq, by reference so that it is read where the
// writer tests it. At f <= 0 every
// output of a frequency is NaN, like f**(1/3): Fe is even in f (s flips sign), so without it f < 0 would give Fe(|f|).

// plain Fp / Fe: the term [P][F] and the inner products [P][F][5] (s|s), (s|c), (c|c), (s|r), (c|r); either may be null
struct FpOut {
  double* terms;
  double* inner;
  // M = [[ss, sc],[sc, cc]], N = [sr, cr]; no f^(-1/3) prefactor: it cancels in every statistic
  __device__ __forceinline__ void put(int p, int64_t f, int64_t F, const double& fq, double ss, double sc, double cc,
                                      double sr, double cr) const {
    double val = term_2x2(ss, sc, cc, sr, cr);
    if (!(fq > 0.0)) val = kNaN();
    if (terms) terms[(size_t)p * F + f] = val;
    if (inner) {
      double* o = inner + ((size_t)p * F + f) * 5;
      o[0] = ss; o[1] = sc; o[2] = cc; o[3] = sr; o[4] = cr;
      if (!(fq > 0.0)) {
#pragma unroll
        for (int k = 0; k < 5; ++k) o[k] = kNaN();
      }
    }
  }
};

// plain Fp / Fe of wide pulsars (DESIGN.md section 5h): what their row-group items write, for row_group_combine_kernel.
// Group 0 of wide pulsar w (meta index first + w) writes (s|s) - b_0, (s|c) - b_0, (c|c) - b_0, (s|r), (c|r) through
// FpOut::put into part [nwide][F][5] at row w; every other item (meta index first + nwide + k) writes its raw b-sums
// b_ss, b_sc, b_cc into b [items - nwide][F][3] at row k. Meta indices below first are whole pulsars.
struct RowGroupOut {
  double* part;
  double* b;
  int first;  // P
  int nwide;
  __device__ __forceinline__ double* part_at(int w, int64_t f, int64_t F) const { return part + ((size_t)w * F + f) * 5; }
  __device__ __forceinline__ double* b_at(int k, int64_t f, int64_t F) const { return b + ((size_t)k * F + f) * 3; }
  // item `item`, frequency f: producer sums a = (sNs, sNc, cNc, s.w, c.w), b-sums of its rows bs
  __device__ __forceinline__ void put(int item, int64_t f, int64_t F, const double& fq, const double (&a)[5],
                                      const double (&bs)[3]) const {
    const int k = item - first;
    if (k < nwide) {
      FpOut{nullptr, part}.put(k, f, F, fq, a[0] - bs[0], a[1] - bs[1], a[2] - bs[2], a[3], a[4]);
    } else {
      double* o = b_at(k - nwide, f, F);
      o[0] = bs[0]; o[1] = bs[1]; o[2] = bs[2];
    }
  }
};

// nmfp stage A, per 32-frequency tile: z'_s, z'_c of the per-draw rows,
// Z [P][nt32][mvpad/4][8][32], and the draw-independent a-terms a_ss, a_sc, a_cc (fixed block removed), a_sr, a_cr,
// A [P][nt32][5][32]
struct NmfpTiles {
  double* Z;
  double* A;
  int mvpad;  // per-draw block width padded to the stage-B tile; rows follow the top padding
  // the z' sin slot of (pulsar p, frequency f, row jr of the padded block); cos is +16. MMA B-fragment order: k-block
  // (jr / 4), column block (4 frequencies), then 16 * {sin, cos} + 4 * (f % 4) + jr % 4 -- what stage B loads
  // without bank conflicts
  __device__ __forceinline__ double* z(int p, int64_t f, int64_t nt32, int jr) const {
    const int fi = (int)(f & 31);
    return Z + ((size_t)p * nt32 + (f >> 5)) * ((size_t)mvpad * 64) +
           (size_t)(((jr >> 2) * 8 + (fi >> 2)) * 32 + 4 * (fi & 3) + (jr & 3));
  }
  __device__ __forceinline__ void put_a(int p, int64_t f, int64_t nt32, double ss, double sc, double cc, double sr,
                                        double cr) const {
    double* o = A + ((size_t)p * nt32 + (f >> 5)) * 160 + (f & 31);
    o[0] = ss; o[32] = sc; o[64] = cc; o[96] = sr; o[128] = cr;
  }
};

// residual batches of R realisations: Fp terms [R][P][F], or (Fe) x = (s|r_k), (c|r_k) as [F][P][R][2] and
// mi = (s|s), (s|c), (c|c) as [F][P][3]; the pointers of the other kind are null
struct ResOut {
  double* terms;
  double* x;
  double* mi;
  int R, P;
  __device__ __forceinline__ void put_m(int p, int64_t f, const double& fq, double ss, double sc, double cc) const {
    if (!mi) return;
    double* o = mi + ((size_t)f * P + p) * 3;
    const bool fpos = fq > 0.0;
    o[0] = fpos ? ss : kNaN();
    o[1] = fpos ? sc : kNaN();
    o[2] = fpos ? cc : kNaN();
  }
  // realisation k: M = [[m00, m01],[m01, m11]], N = [sr, cr]
  __device__ __forceinline__ void put(int k, int p, int64_t f, int64_t F, const double& fq, double m00, double m01,
                                      double m11, double sr, double cr) const {
    const bool fpos = fq > 0.0;
    if (x) {
      *reinterpret_cast<double2*>(x + (((size_t)f * P + p) * R + k) * 2) =
          fpos ? make_double2(sr, cr) : make_double2(kNaN(), kNaN());
      return;
    }
    double val = term_2x2(m00, m01, m11, sr, cr);
    if (!fpos) val = kNaN();
    terms[((size_t)k * P + p) * F + f] = val;
  }
};

// ---- sweep launchers (fp_sweep*.cu), each with the output block of its mode ----------------
// with wide pulsars, also their row-group combine into `out`, through the pack's row-group scratch
// (pk->rg_doubles_per_freq() doubles per frequency)
int launch_fp_sweep(const fastfp_pack* pk, const double* d_freqs, int64_t F, const FpOut& out, cudaStream_t st,
                    bool rest_only = false);
int launch_fp_sweep(const fastfp_pack* pk, const double* d_freqs, int64_t F, const NmfpTiles& out, cudaStream_t st,
                    bool rest_only = false);
// residual batches: the sweep over the pack's residual packets (fp_sweep.cu)
int launch_fp_sweep_res(const fastfp_pack* pk, const double* d_freqs, int64_t F, const ResOut& out, cudaStream_t st);
// the pulsar sum of each row of [R][P][F] terms into out[k * ld + f] (R = 1: the terms of a plain sweep)
int launch_reduce_terms_rows(const double* d_terms, int R, int P, int64_t F, double* d_out, int64_t ld,
                             cudaStream_t st);
// fp_sweep_i8.cu
bool i8_eligible(const fastfp_pack* pk);
int build_i8_planes(fastfp_pack* pk, cudaStream_t st);
int run_i8_peak(int kind, int iters, double* tops, double* ms);
int launch_fp_sweep_i8(const fastfp_pack* pk, const double* d_freqs, int64_t F, const FpOut& out, cudaStream_t st);
int launch_fp_sweep_i8(const fastfp_pack* pk, const double* d_freqs, int64_t F, const NmfpTiles& out, cudaStream_t st);
// the sweep on the path(s) the pack is set to: the tensor kernel for the pulsars it takes, the fp64 kernel for the rest
template <class Out>  // FpOut or NmfpTiles
int launch_sweep(const fastfp_pack* pk, const double* d_freqs, int64_t F, const Out& out, cudaStream_t st) {
  if (!pk->use_i8()) return launch_fp_sweep(pk, d_freqs, F, out, st);
  if (int rc = launch_fp_sweep_i8(pk, d_freqs, F, out, st)) return rc;
  return pk->i8_all() ? 0 : launch_fp_sweep(pk, d_freqs, F, out, st, true);
}

}  // namespace ffp
