// extern "C" entry points of libfastfp_b200.so (declared in include/fastfp_b200.h).
#include <algorithm>
#include <cmath>
#include <cstring>

#include "../../include/fastfp_b200.h"
#include "ffp_internal.cuh"

namespace ffp {

std::atomic<int64_t> g_launches{0};
std::atomic<int64_t> g_device_bytes{0};
static thread_local std::string t_err;

void set_error(const std::string& msg) { t_err = msg; }
int cuda_fail(cudaError_t e, const char* what) {
  t_err = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what;
  return FASTFP_ERR_CUDA;
}

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; }
    if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};


// nmfp.cu
int nmfp_pack_finish(fastfp_pack* pk, const double* d_toas, const double* d_res,
                     const double* d_Nvec, const double* d_T, const double* d_TNT,
                     const double* d_phiinv_fix, cudaStream_t st, const BlockNDev* bn = nullptr);
int nmfp_sweep_impl(const fastfp_pack* pk, const double* d_freqs, int64_t F,
                    const double* d_phiinv_var, int64_t D, double* d_out, cudaStream_t st);
int nmfp_stage_a_impl(const fastfp_pack* pk, const double* d_freqs, int64_t F, double* dZ, double* dA, cudaStream_t st);
int nmfp_stage_b_only(const fastfp_pack* pk, const double* d_freqs, int64_t F, const double* dZ, const double* dA,
                      int nt_blk, const double* d_phiinv_var, int64_t D, double* d_out, cudaStream_t st);
int powerlaw_phiinv_impl(const fastfp_pack* pk, const double* const* Ffreqs, const double* log10_A,
                         const double* gamma, int64_t D, const double* curn_Ffreqs, int64_t ncurn,
                         const double* curn_log10_A, const double* curn_gamma, double* out,
                         cudaStream_t st);

static int pack_layout(fastfp_pack* pk, int P, const int64_t* n, const int64_t* m,
                       const int64_t* m_fix, const double* const* toas, bool blockn = false) {
  pk->P = P;
  pk->meta.resize(P);
  int64_t L_off = 0, raw_off = 0, T_off = 0, dm_off = 0;
  int var_off = 0;
  pk->ecorr = blockn;
  PacketLayout lay;
  for (int p = 0; p < P; ++p) {
    if (n[p] < 1 || m[p] < 1 || n[p] > 0x7fffff00LL) {
      set_error("pulsar " + std::to_string(p) + ": n and m must be positive");
      return FASTFP_ERR_INVALID;
    }
    PulsarMeta& pm = pk->meta[p];
    pm.n = (int)n[p];
    // bases wider than one work item: row groups, placed after the loop (diagonal-N Fp packs only)
    const bool grouped = !blockn && !m_fix && m[p] > MAX_M && m[p] <= MAX_M_WIDE;
    if (!grouped && (m[p] > MAX_M || !lay.place(p, sweep_rows((int)m[p], 0, blockn), &pm))) {
      set_error("pulsar " + std::to_string(p) + ": basis width m=" + std::to_string(m[p]) +
                (blockn ? " exceeds the block-N maximum " + std::to_string(MAX_M - 8) + " (the widest kernel has " +
                              std::to_string(MAX_M) + " rows, 8 of them hold the epoch slots)"
                 : m_fix ? " exceeds the noise-marginalised maximum " + std::to_string(MAX_M)
                         : " exceeds the supported maximum " + std::to_string(MAX_M_WIDE)));
      return FASTFP_ERR_UNSUPPORTED;
    }
    pm.m = (int)m[p];
    pm.L_off = L_off;
    pm.raw_off = raw_off;
    pm.T_off = T_off;
    pm.mfix = m_fix ? (int)m_fix[p] : pm.m;
    pm.mvar = pm.m - pm.mfix;
    if (pm.mfix < 0 || pm.mvar < 0) {
      set_error("pulsar " + std::to_string(p) + ": m_fix out of range");
      return FASTFP_ERR_INVALID;
    }
    pm.var_off = var_off;
    pm.dm_off = dm_off;
    if (blockn && pm.n % pm.ci != 0) {
      set_error("block-N pack: the TOA count must be a multiple of the chunk size (fastfp_sweep_chunk_toas)");
      return FASTFP_ERR_INVALID;
    }
    dm_off += pm.nch;
    pm.tabs_max = 0.0;
    if (!toas[p]) { set_error("null toas"); return FASTFP_ERR_INVALID; }
    for (int64_t i = 0; i < n[p]; ++i) {
      const double a = std::fabs(toas[p][i]);
      if (!(a <= 1.7e308)) { pm.tabs_max = INFINITY; break; }
      if (a > pm.tabs_max) pm.tabs_max = a;
    }
    var_off += pm.mvar;
    pk->mvar_max = std::max(pk->mvar_max, pm.mvar);
    L_off += (int64_t)pm.m * pm.m;
    raw_off += pm.n;
    T_off += (int64_t)pm.n * pm.m;
  }
  pk->mvar_total = var_off;
  // row groups (DESIGN.md section 5h): one work item per group, meta indices P ..., each placed like a pulsar of its
  // rows: group 0 of every wide pulsar first, then the other groups pulsar by pulsar
  std::vector<int> wide;
  for (int p = 0; p < P; ++p)
    if (row_groups(pk->meta[p].m) > 1) wide.insert(wide.end(), {p, 0, 0, row_groups(pk->meta[p].m)});
  for (int pass = 0; pass < 2; ++pass)
    for (size_t w = 0; w < wide.size(); w += RG_WIDE) {
      const PulsarMeta& pm = pk->meta[wide[w]];
      wide[w + 1 + pass] = P + (int)pk->items.size();
      for (int k = pass; k < (pass ? wide[w + 3] : 1); ++k) {
        PulsarMeta it = pm;
        it.m = it.mfix = row_group_start(pm.m, k + 1) - row_group_start(pm.m, k);
        it.mvar = 0;
        lay.place(P + (int)pk->items.size(), sweep_rows(it.m, 0, false), &it);  // <= 288 rows: always placed
        pk->items.push_back(it);
      }
    }
  pk->n_wide = (int)wide.size() / RG_WIDE;
  const int nmeta = P + (int)pk->items.size();
  PackCore& c = pk->core;
  FFP_CUDA(dev_alloc(&c.meta, (size_t)nmeta));
  FFP_CUDA(cudaMemcpy(c.meta.get(), pk->meta.data(), sizeof(PulsarMeta) * P, cudaMemcpyHostToDevice));
  if (pk->n_wide) {
    FFP_CUDA(cudaMemcpy(c.meta.get() + P, pk->items.data(), sizeof(PulsarMeta) * pk->items.size(),
                        cudaMemcpyHostToDevice));
    FFP_CUDA(dev_alloc(&c.wide, wide.size()));
    FFP_CUDA(cudaMemcpy(c.wide.get(), wide.data(), sizeof(int) * wide.size(), cudaMemcpyHostToDevice));
  }
  FFP_CUDA(dev_alloc(&c.packets, (size_t)lay.size));
  FFP_CUDA(dev_alloc(&c.L, (size_t)L_off));
  FFP_CUDA(dev_alloc(&c.info, (size_t)P));
  FFP_CUDA(cudaMemset(c.info.get(), 0, sizeof(int) * P));
  FFP_CUDA(cudaDeviceGetAttribute(&pk->num_sms, cudaDevAttrMultiProcessorCount, pk->device));
  const size_t slab_doubles = (size_t)CTAS_PER_SM * pk->num_sms * sweep_max_slab_doubles();
  FFP_CUDA(dev_alloc(&c.slab, slab_doubles));
  FFP_CUDA(dev_alloc(&c.counter, 1));
  pk->bytes = lay.size * 8 + L_off * 8 + (int64_t)sizeof(PulsarMeta) * nmeta + (int64_t)slab_doubles * 8 +
              (int64_t)sizeof(int) * wide.size();
  return lay.upload(&pk->groups);
}

// which: 0 = length n_p, 1 = n_p*m_p (T), 2 = m_p*m_p
static int64_t ragged_count(const PulsarMeta& pm, int which) {
  return which == 0 ? pm.n : which == 1 ? (int64_t)pm.n * pm.m : (int64_t)pm.m * pm.m;
}

// the per-pulsar arrays src[p] back to back into dst
static int upload_ragged(double* dst, const double* const* src, const fastfp_pack* pk, int which, cudaStream_t st) {
  int64_t off = 0;
  for (int p = 0; p < pk->P; ++p) {
    const int64_t cnt = ragged_count(pk->meta[p], which);
    if (!src[p]) { set_error("null per-pulsar array"); return FASTFP_ERR_INVALID; }
    FFP_CUDA(cudaMemcpyAsync(dst + off, src[p], (size_t)cnt * 8, cudaMemcpyHostToDevice, st));
    off += cnt;
  }
  return 0;
}

// upload_ragged into a new staging buffer
static int stage_ragged(DeviceBuf<double>* dst, const double* const* src, const fastfp_pack* pk, int which,
                        cudaStream_t st) {
  int64_t total = 0;
  for (auto& pm : pk->meta) total += ragged_count(pm, which);
  FFP_CUDA(dev_alloc(dst, (size_t)total));
  return upload_ragged(dst->get(), src, pk, which, st);
}

// sum_i 1/N_i per pulsar in extended precision (the tensor sweep derives c N^-1 c from s N^-1 s with it)
static void set_ninv_sums(fastfp_pack* pk, const double* const* Nvecs) {
  for (int p = 0; p < pk->P; ++p) {
    long double acc = 0.0L;
    for (int i = 0; i < pk->meta[p].n; ++i) acc += 1.0L / (long double)Nvecs[p][i];
    pk->meta[p].ninv_sum = (double)acc;
  }
}

static void pack_free(fastfp_pack* pk) {
  if (!pk) return;
  DeviceGuard g(pk->device);
  delete pk;  // the pack owns all its memory: released while its device is current
}

struct BlockNHost {  // host side arrays of a block-diagonal N (fastfp_pack_create_blockn)
  const double* const* res_w;
  const int32_t* const* slot_idx;
  const double* const* slot_val;
  const unsigned char* const* done_mask;
};

// block-N slot indices into a new staging buffer, the per-chunk slot masks into the pack
static int stage_slots(fastfp_pack* pk, const BlockNHost& bn, DeviceBuf<int>* d_sidx, cudaStream_t st) {
  int64_t ntot = 0, nchtot = 0;
  for (auto& pm : pk->meta) { ntot += pm.n; nchtot += pm.nch; }
  FFP_CUDA(dev_alloc(d_sidx, (size_t)ntot));
  FFP_CUDA(dev_alloc(&pk->core.done_mask, (size_t)nchtot));
  for (int p = 0; p < pk->P; ++p) {
    const PulsarMeta& pm = pk->meta[p];
    if (!bn.slot_idx[p] || !bn.done_mask[p]) { set_error("null slot array"); return FASTFP_ERR_INVALID; }
    FFP_CUDA(cudaMemcpyAsync(d_sidx->get() + pm.raw_off, bn.slot_idx[p], (size_t)pm.n * sizeof(int),
                             cudaMemcpyHostToDevice, st));
    FFP_CUDA(cudaMemcpyAsync(pk->core.done_mask.get() + pm.dm_off, bn.done_mask[p], (size_t)pm.nch,
                             cudaMemcpyHostToDevice, st));
  }
  return 0;
}

// The one pack builder behind the three constructors. mats are the sigmas of a plain-Fp pack (m_fix null) or the TNTs
// of an nmfp pack (m_fix / phiinv_fix: the draw-independent leading columns and their prior). bn null: diagonal N.
static int build_pack(int device, int P, const int64_t* n, const int64_t* m, const double* const* toas,
                      const double* const* residuals, const double* const* Nvecs, const double* const* Ts,
                      const double* const* mats, const int64_t* m_fix, const double* const* phiinv_fix,
                      const BlockNHost* bn, void* stream, fastfp_pack_t** out) {
  *out = nullptr;
  DeviceGuard g(device);
  if (!g.ok) { set_error("cannot select CUDA device " + std::to_string(device)); return FASTFP_ERR_CUDA; }
  cudaStream_t st = (cudaStream_t)stream;
  fastfp_pack* pk = new fastfp_pack();
  pk->device = device;
  pk->nmfp = m_fix != nullptr;
  int rc = pack_layout(pk, P, n, m, m_fix, toas, bn != nullptr);
  DeviceBuf<double> d_toas, d_res, d_Nvec, d_T, d_mat, d_pf, d_resw, d_sval;
  DeviceBuf<int> d_sidx;
  if (!rc) rc = stage_ragged(&d_toas, toas, pk, 0, st);
  if (!rc) rc = stage_ragged(&d_res, residuals, pk, 0, st);
  if (!rc) rc = stage_ragged(&d_Nvec, Nvecs, pk, 0, st);
  if (!rc) rc = stage_ragged(&d_T, Ts, pk, 1, st);
  if (!rc && bn) rc = stage_ragged(&d_resw, bn->res_w, pk, 0, st);
  if (!rc && bn) rc = stage_ragged(&d_sval, bn->slot_val, pk, 0, st);
  if (!rc && bn) rc = stage_slots(pk, *bn, &d_sidx, st);
  const BlockNDev bnd{d_resw.get(), d_sidx.get(), d_sval.get()};
  const BlockNDev* bnp = bn ? &bnd : nullptr;
  if (!rc && !bn) set_ninv_sums(pk, Nvecs);  // only the tensor sweep reads them, and it takes no block-N pack
  if (!rc && !pk->nmfp) {
    rc = upload_ragged(pk->core.L.get(), mats, pk, 2, st);  // sigmas, into the factor buffer pack_layout allocated
    if (!rc) rc = launch_fp_precompute(pk, d_toas.get(), d_res.get(), d_Nvec.get(), d_T.get(), st, nullptr, bnp);
    if (!rc) rc = build_i8_planes(pk, st);  // digit planes for the pulsars the tensor sweep takes (none with block-N)
  } else if (!rc) {
    rc = stage_ragged(&d_mat, mats, pk, 2, st);  // TNTs
    if (!rc) {
      // fixed phiinv: (P, MAX_M) padded
      std::vector<double> pf((size_t)P * MAX_M, 0.0);
      for (int p = 0; p < P; ++p)
        for (int j = 0; j < pk->meta[p].mfix; ++j) pf[(size_t)p * MAX_M + j] = phiinv_fix[p][j];
      cudaError_t e = dev_alloc(&d_pf, pf.size());
      if (e == cudaSuccess) e = cudaMemcpy(d_pf.get(), pf.data(), pf.size() * 8, cudaMemcpyHostToDevice);
      if (e != cudaSuccess) rc = cuda_fail(e, "upload phiinv_fix");
    }
    if (!rc) rc = nmfp_pack_finish(pk, d_toas.get(), d_res.get(), d_Nvec.get(), d_T.get(), d_mat.get(), d_pf.get(), st, bnp);
  }
  cudaStreamSynchronize(st);  // the staging buffers are released on return, after the work that reads them
  if (rc) { pack_free(pk); return rc; }
  *out = pk;
  return FASTFP_OK;
}

// The start and end of every call that runs work on a pack. While it lives the pack's device is current; select()
// reports FASTFP_ERR_CUDA if it could not be made so. stage() also resolves the device addresses of the F frequencies
// (the caller's pointer, or the host array copied into pk->freqs) and of the nout result doubles (the caller's pointer,
// or the pack-owned buffer *buf that finish() copies back to host memory).
struct PackCall {
  const fastfp_pack* pk;
  cudaStream_t st;
  DeviceGuard dev;
  PackCall(const fastfp_pack* p, void* stream) : pk(p), st((cudaStream_t)stream), dev(p->device) {}
  int select() const {
    if (dev.ok) return FASTFP_OK;
    set_error("cannot select CUDA device " + std::to_string(pk->device));
    return FASTFP_ERR_CUDA;
  }
  int stage(const double* freqs, int64_t F, double* out, int64_t nout, int flags, const double** d_freqs,
            double** d_out, Scratch<double>* buf) const {
    if (int rc = select()) return rc;
    *d_freqs = freqs;
    if (!(flags & FASTFP_FREQS_ON_DEVICE)) {
      if (int rc = pk->freqs.grow(F)) return rc;
      FFP_CUDA(cudaMemcpyAsync(pk->freqs.get(), freqs, (size_t)F * 8, cudaMemcpyHostToDevice, st));
      *d_freqs = pk->freqs.get();
    }
    *d_out = out;
    if (!(flags & FASTFP_OUT_ON_DEVICE)) {
      if (int rc = buf->grow(nout)) return rc;
      *d_out = buf->get();
    }
    return FASTFP_OK;
  }
  // The antenna patterns fplus / fcross, n doubles each, into the scratch at d_fp / d_fx. They are read from memory the
  // caller owns and may change or free once the call returns, so every Fe call synchronises before it returns, even
  // when its outputs stay on the device.
  int upload_sky(const double* fplus, const double* fcross, int64_t n, double* d_fp, double* d_fx) const {
    FFP_CUDA(cudaMemcpyAsync(d_fp, fplus, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    FFP_CUDA(cudaMemcpyAsync(d_fx, fcross, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    return FASTFP_OK;
  }
  // Copies the n result doubles d_out (and the n indices d_idx, if the call has them) to the caller's host memory
  // unless FASTFP_OUT_ON_DEVICE says they stay where they are, then waits for the stream: always after such a copy,
  // and with outputs on the device only if `always`.
  int finish(int flags, int64_t n, double* out, const double* d_out, bool always, int64_t* idx = nullptr,
             const int64_t* d_idx = nullptr) const {
    const bool to_host = !(flags & FASTFP_OUT_ON_DEVICE);
    if (to_host) {
      FFP_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
      if (idx) FFP_CUDA(cudaMemcpyAsync(idx, d_idx, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    }
    if (to_host || always) FFP_CUDA(cudaStreamSynchronize(st));
    return FASTFP_OK;
  }
};

// Frequencies are processed in batches so the per-batch scratch (terms or inner products) stays bounded.
static const int64_t kTermBudgetDoubles = 1LL << 27;  // 1 GiB

// frequencies per batch of a sweep whose scratch holds doubles_per_freq doubles per frequency: at least 1024
static int64_t freq_batch(int64_t F, int64_t doubles_per_freq) {
  return std::max<int64_t>(1024, std::min<int64_t>(F, kTermBudgetDoubles / doubles_per_freq));
}

// Offsets of the regions of one scratch buffer, taken in the order they are laid out, in 8-byte slots (doubles or
// int64); total is what the buffer must hold.
struct ScratchLayout {
  int64_t total = 0;
  int64_t take(int64_t n) {
    const int64_t at = total;
    total += n;
    return at;
  }
};

// The limit of a residual batch: every pulsar takes sweep_rows(m, R, blockn) of the kernel's MAX_M G rows, so the widest
// one bounds R. FASTFP_ERR_UNSUPPORTED with a message that names the limit and that pulsar for an R above it.
static int check_res_limit(const fastfp_pack* pk, int64_t R, const char* fn) {
  for (int p = 0; p < pk->P && R > 0; ++p)  // R == 0 releases a set, which any pack may do
    if (pk->meta[p].m > MAX_M) {
      set_error(std::string(fn) + ": pulsar " + std::to_string(p) + " has a basis wider than " + std::to_string(MAX_M) +
                " columns (m = " + std::to_string(pk->meta[p].m) + "); residual batches take bases up to " +
                std::to_string(MAX_M) + " columns");
      return FASTFP_ERR_UNSUPPORTED;
    }
  int wide = 0;
  for (int p = 0; p < pk->P; ++p)
    if (pk->meta[p].m > pk->meta[wide].m) wide = p;
  const int64_t rmax = MAX_M - sweep_rows(pk->meta[wide].m, 0, pk->ecorr);
  if (R <= rmax) return FASTFP_OK;
  set_error(std::string(fn) + ": R = " + std::to_string(R) + " exceeds the limit of " + std::to_string(rmax) +
            " for this pack: its widest pulsar " + std::to_string(wide) + " (m = " + std::to_string(pk->meta[wide].m) +
            (pk->ecorr ? ") and the 8 epoch-slot rows leave " : ") leaves ") + std::to_string(rmax) +
            " of the sweep kernel's " + std::to_string(MAX_M) + " G rows");
  return FASTFP_ERR_UNSUPPORTED;
}

// Replaces the pack's residual batch with the R realisations of h (R == 0: none), once the sweeps queued on the stream,
// which may still read the previous set, are done
static int replace_res(fastfp_pack* pk, int64_t R, const ResHost& h, void* stream, const SimHost* sim = nullptr) {
  PackCall c(pk, stream);
  if (int rc = c.select()) return rc;
  FFP_CUDA(cudaStreamSynchronize(c.st));
  pk->res = {};
  if (R == 0) return FASTFP_OK;
  return build_res_packets(pk, R, h, c.st, sim);
}

// The arguments both simulate entry points share (fastfp_pack_simulate_residuals*): FASTFP_ERR_INVALID for a negative
// seed or first index, a signal given by half, an unknown flag, or a prior that is not finite and >= 0
static int check_sim_args(const fastfp_pack* pk, int64_t R, int64_t seed, int64_t first, const double* const* phiinv,
                          const double* sig_freq, const double* sig_amp, int flags, const char* fn) {
  if (seed < 0 || first < 0 || first > INT64_MAX - R || (!sig_freq != !sig_amp) || (flags & ~FASTFP_SIM_NO_NOISE)) {
    set_error(std::string(fn) + ": seed and first must be >= 0, sig_freq and sig_amp both given or both NULL, and "
              "flags 0 or FASTFP_SIM_NO_NOISE");
    return FASTFP_ERR_INVALID;
  }
  for (int p = 0; p < pk->P && R > 0; ++p) {
    if (!phiinv[p]) { set_error(std::string(fn) + ": null per-pulsar array"); return FASTFP_ERR_INVALID; }
    for (int j = 0; j < pk->meta[p].m; ++j) {
      if (!(phiinv[p][j] >= 0.0) || !std::isfinite(phiinv[p][j])) {
        set_error(std::string(fn) + ": pulsar " + std::to_string(p) + ": phiinv[" + std::to_string(j) +
                  "] must be finite and >= 0");
        return FASTFP_ERR_INVALID;
      }
    }
  }
  return FASTFP_OK;
}

}  // namespace ffp

using namespace ffp;

extern "C" {

const char* fastfp_last_error(void) { return t_err.c_str(); }
int fastfp_version(void) { return 100; }
int fastfp_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}
int64_t fastfp_kernel_launches(void) { return g_launches.load(); }
int64_t fastfp_device_bytes(void) { return g_device_bytes.load(); }

int fastfp_pack_create(int device, int P, const int64_t* n, const int64_t* m,
                       const double* const* toas, const double* const* residuals,
                       const double* const* Nvecs, const double* const* Ts,
                       const double* const* sigmas, void* stream, fastfp_pack_t** out) {
  if (!out || P < 1 || !n || !m || !toas || !residuals || !Nvecs || !Ts || !sigmas) {
    set_error("fastfp_pack_create: null argument or P < 1");
    return FASTFP_ERR_INVALID;
  }
  return build_pack(device, P, n, m, toas, residuals, Nvecs, Ts, sigmas, nullptr, nullptr, nullptr, stream, out);
}

int fastfp_pack_set_path(fastfp_pack_t* pk, int path) {
  if (!pk || path < FASTFP_PATH_AUTO || path > FASTFP_PATH_MIXED) {
    set_error("fastfp_pack_set_path: invalid argument");
    return FASTFP_ERR_INVALID;
  }
  if (path == FASTFP_PATH_I8 && !(pk->i8.ok && pk->i8_all())) {
    set_error("fastfp_pack_set_path: not every pulsar of this pack has INT8 digit planes (block-diagonal N, m > 639, "
              "n > 16384 or non-finite data); FASTFP_PATH_MIXED sweeps those on the fp64 kernel");
    return FASTFP_ERR_UNSUPPORTED;
  }
  if (path == FASTFP_PATH_MIXED && !pk->i8.ok) {
    set_error("fastfp_pack_set_path: no pulsar of this pack has INT8 digit planes");
    return FASTFP_ERR_UNSUPPORTED;
  }
  pk->path = path;
  return FASTFP_OK;
}

int fastfp_pack_path(const fastfp_pack_t* pk) {
  if (!pk) return FASTFP_ERR_INVALID;
  return pk->use_i8() ? (pk->i8_all() ? FASTFP_PATH_I8 : FASTFP_PATH_MIXED) : FASTFP_PATH_FP64;
}

int fastfp_nmfp_pack_create(int device, int P, const int64_t* n, const int64_t* m,
                            const double* const* toas, const double* const* residuals,
                            const double* const* Nvecs, const double* const* Ts,
                            const double* const* TNTs, const int64_t* m_fix,
                            const double* const* phiinv_fix, void* stream, fastfp_pack_t** out) {
  if (!out || P < 1 || !n || !m || !toas || !residuals || !Nvecs || !Ts || !TNTs || !m_fix ||
      !phiinv_fix) {
    set_error("fastfp_nmfp_pack_create: null argument or P < 1");
    return FASTFP_ERR_INVALID;
  }
  return build_pack(device, P, n, m, toas, residuals, Nvecs, Ts, TNTs, m_fix, phiinv_fix, nullptr, stream, out);
}

int fastfp_sweep_chunk_toas(int64_t m, int blockn) {
  KernelCfg kc{};
  if (m < 1 || m > MAX_M || !sweep_config(sweep_rows((int)m, 0, blockn != 0), &kc)) return 0;
  return kc.ci;
}

int fastfp_row_groups(int64_t m, int64_t* starts) {
  if (m < 1 || m > MAX_M_WIDE) return 0;
  const int g = row_groups((int)m);
  for (int k = 0; starts && k <= g; ++k) starts[k] = row_group_start((int)m, k);
  return g;
}

int fastfp_pack_create_blockn(int device, int P, const int64_t* n, const int64_t* m,
                              const double* const* toas, const double* const* residuals,
                              const double* const* residuals_w, const double* const* Nvecs,
                              const double* const* Ts, const double* const* mats,
                              const int32_t* const* slot_idx, const double* const* slot_val,
                              const unsigned char* const* done_mask, const int64_t* m_fix,
                              const double* const* phiinv_fix, void* stream, fastfp_pack_t** out) {
  if (!out || P < 1 || !n || !m || !toas || !residuals || !residuals_w || !Nvecs || !Ts || !mats ||
      !slot_idx || !slot_val || !done_mask || (m_fix && !phiinv_fix)) {
    set_error("fastfp_pack_create_blockn: null argument or P < 1");
    return FASTFP_ERR_INVALID;
  }
  const BlockNHost bn{residuals_w, slot_idx, slot_val, done_mask};
  return build_pack(device, P, n, m, toas, residuals, Nvecs, Ts, mats, m_fix, phiinv_fix, &bn, stream, out);
}

void fastfp_pack_destroy(fastfp_pack_t* pack) { pack_free(pack); }
int64_t fastfp_pack_bytes(const fastfp_pack_t* pack) {
  return pack ? pack->bytes + pack->res.bytes + pack->rg.cap * 8 : 0;
}
int fastfp_pack_num_pulsars(const fastfp_pack_t* pack) { return pack ? pack->P : 0; }
int64_t fastfp_pack_mvar_total(const fastfp_pack_t* pack) { return pack ? pack->mvar_total : 0; }
int fastfp_pack_factor_info(const fastfp_pack_t* pack, int32_t* info) {
  if (!pack) { set_error("fastfp_pack_factor_info: null pack"); return FASTFP_ERR_INVALID; }
  int bad = 0;
  for (int p = 0; p < pack->P; ++p) {
    const int v = p < (int)pack->info.size() ? pack->info[p] : 0;
    if (info) info[p] = v;
    bad += v != 0;
  }
  return bad;
}

static int fp_run(const fastfp_pack* pk, const double* freqs, int64_t F, double* out, int flags,
                  void* stream, bool want_terms) {
  if (!pk || (F > 0 && (!freqs || !out)) || F < 0) {
    set_error("fastfp_fp_sweep: null argument or negative F");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) { set_error("this pack was built for nmfp; use fastfp_nmfp_sweep"); return FASTFP_ERR_INVALID; }
  if (F == 0) return FASTFP_OK;
  const int P = pk->P;
  const int64_t nout = want_terms ? (int64_t)P * F : F;
  // the batches bound the terms scratch and, with wide pulsars, the row-group scratch; the terms of a call go straight
  // to its output unless a pack with wide pulsars needs more than one batch for them
  const int64_t FB = freq_batch(F, P + pk->rg_doubles_per_freq());
  const bool direct = want_terms && (FB >= F || !pk->n_wide);
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_out;
  if (int rc = c.stage(freqs, F, out, nout, flags, &d_freqs, &d_out, direct ? &pk->terms : &pk->out)) return rc;
  if (direct) {
    if (int rc = launch_sweep(pk, d_freqs, F, FpOut{d_out, nullptr}, c.st)) return rc;
  } else {
    if (int rc = pk->terms.grow((int64_t)P * std::min(FB, F))) return rc;
    for (int64_t lo = 0; lo < F; lo += FB) {
      const int64_t fb = std::min(FB, F - lo);
      if (int rc = launch_sweep(pk, d_freqs + lo, fb, FpOut{pk->terms.get(), nullptr}, c.st)) return rc;
      if (want_terms) {
        FFP_CUDA(cudaMemcpy2DAsync(d_out + lo, (size_t)F * 8, pk->terms.get(), (size_t)fb * 8, (size_t)fb * 8,
                                   (size_t)P, cudaMemcpyDeviceToDevice, c.st));
      } else if (int rc = launch_reduce_terms_rows(pk->terms.get(), 1, P, fb, d_out + lo, F, c.st)) {
        return rc;
      }
    }
  }
  return c.finish(flags, nout, out, d_out, false);
}

int fastfp_fp_sweep(const fastfp_pack_t* pack, const double* freqs, int64_t F, double* out,
                    int flags, void* stream) {
  return fp_run(pack, freqs, F, out, flags, stream, false);
}
int fastfp_fp_terms(const fastfp_pack_t* pack, const double* freqs, int64_t F, double* terms,
                    int flags, void* stream) {
  return fp_run(pack, freqs, F, terms, flags, stream, true);
}

// Residual batches (DESIGN.md section 5d): R realisations of the residuals as extra G rows of the fp64 kernel
int fastfp_pack_set_residuals(fastfp_pack_t* pk, int64_t R, const double* const* residuals, void* stream) {
  if (!pk || R < 0 || (R > 0 && !residuals)) {
    set_error("fastfp_pack_set_residuals: null argument or negative R");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) { set_error("fastfp_pack_set_residuals needs a plain-Fp pack (fastfp_pack_create)"); return FASTFP_ERR_INVALID; }
  if (pk->ecorr) {
    set_error("fastfp_pack_set_residuals: a block-diagonal N pack takes its realisations in its own TOA layout "
              "(fastfp_pack_set_residuals_blockn)");
    return FASTFP_ERR_UNSUPPORTED;
  }
  std::vector<int64_t> n(pk->P);
  for (int p = 0; p < pk->P; ++p) {
    if (R > 0 && !residuals[p]) { set_error("fastfp_pack_set_residuals: null per-pulsar array"); return FASTFP_ERR_INVALID; }
    n[p] = pk->meta[p].n;
  }
  if (int rc = check_res_limit(pk, R, "fastfp_pack_set_residuals")) return rc;
  return replace_res(pk, R, {n.data(), residuals, residuals, nullptr, nullptr, nullptr}, stream);
}

// Residual batches of a block-diagonal N pack: the realisations in the TOA layout of the residual kernel's chunk size
int fastfp_pack_set_residuals_blockn(fastfp_pack_t* pk, int64_t R, const int64_t* n, const double* const* residuals,
                                     const double* const* residuals_w, const int32_t* const* slot_idx,
                                     const double* const* slot_val, const unsigned char* const* done_mask,
                                     void* stream) {
  if (!pk || R < 0 || (R > 0 && (!n || !residuals || !residuals_w || !slot_idx || !slot_val || !done_mask))) {
    set_error("fastfp_pack_set_residuals_blockn: null argument or negative R");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) {
    set_error("fastfp_pack_set_residuals_blockn needs a plain-Fp pack (fastfp_pack_create_blockn without m_fix)");
    return FASTFP_ERR_INVALID;
  }
  if (!pk->ecorr) {
    set_error("fastfp_pack_set_residuals_blockn needs a block-diagonal N pack; a diagonal-N pack takes "
              "fastfp_pack_set_residuals");
    return FASTFP_ERR_INVALID;
  }
  if (int rc = check_res_limit(pk, R, "fastfp_pack_set_residuals_blockn")) return rc;
  for (int p = 0; p < pk->P && R > 0; ++p) {
    if (!residuals[p] || !residuals_w[p] || !slot_idx[p] || !slot_val[p] || !done_mask[p]) {
      set_error("fastfp_pack_set_residuals_blockn: null per-pulsar array");
      return FASTFP_ERR_INVALID;
    }
    KernelCfg kc{};
    if (!sweep_config(sweep_rows(pk->meta[p].m, R, true), &kc) || n[p] < 1 || n[p] > 0x7fffff00LL ||
        n[p] % kc.ci != 0) {
      set_error("fastfp_pack_set_residuals_blockn: pulsar " + std::to_string(p) + ": the TOA count " +
                std::to_string(n[p]) + " of the residual layout must be a positive multiple of its chunk size " +
                std::to_string(kc.ci) + " (fastfp_sweep_chunk_toas(roundup8(m) + roundup8(R), 1))");
      return FASTFP_ERR_INVALID;
    }
  }
  return replace_res(pk, R, {n, residuals, residuals_w, slot_idx, slot_val, done_mask}, stream);
}

// Residual batches drawn on the device (DESIGN.md section 5g): the staging that set_residuals fills from the host is
// filled by sim_noise_kernel, and sim_basis_kernel adds the basis draw between G n and w
int fastfp_pack_simulate_residuals(fastfp_pack_t* pk, int64_t R, int64_t seed, int64_t first,
                                   const double* const* phiinv, const double* sig_freq, const double* sig_amp,
                                   int flags, void* stream) {
  if (!pk || R < 0 || (R > 0 && !phiinv)) {
    set_error("fastfp_pack_simulate_residuals: null argument or negative R");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) {
    set_error("fastfp_pack_simulate_residuals needs a plain-Fp pack (fastfp_pack_create)");
    return FASTFP_ERR_INVALID;
  }
  if (pk->ecorr) {
    set_error("fastfp_pack_simulate_residuals: a block-diagonal N pack takes its realisations in its own TOA layout "
              "(fastfp_pack_simulate_residuals_blockn)");
    return FASTFP_ERR_UNSUPPORTED;
  }
  const char* fn = "fastfp_pack_simulate_residuals";
  if (int rc = check_sim_args(pk, R, seed, first, phiinv, sig_freq, sig_amp, flags, fn)) return rc;
  if (int rc = check_res_limit(pk, R, fn)) return rc;
  std::vector<int64_t> n(pk->P);
  for (int p = 0; p < pk->P; ++p) n[p] = pk->meta[p].n;
  const SimHost sim{seed, first, !(flags & FASTFP_SIM_NO_NOISE), phiinv, sig_freq, sig_amp,
                    nullptr, nullptr, nullptr, nullptr};
  return replace_res(pk, R, {n.data(), nullptr, nullptr, nullptr, nullptr, nullptr}, stream, &sim);
}

int fastfp_pack_simulate_residuals_blockn(fastfp_pack_t* pk, int64_t R, int64_t seed, int64_t first,
                                          const double* const* phiinv, const double* sig_freq, const double* sig_amp,
                                          const int64_t* n, const int32_t* const* slot_idx,
                                          const double* const* slot_val, const unsigned char* const* done_mask,
                                          const int32_t* const* toa_index, const int32_t* const* epoch,
                                          const double* const* sqrt_j, const double* const* beta, int flags,
                                          void* stream) {
  if (!pk || R < 0 ||
      (R > 0 && (!phiinv || !n || !slot_idx || !slot_val || !done_mask || !toa_index || !epoch || !sqrt_j || !beta))) {
    set_error("fastfp_pack_simulate_residuals_blockn: null argument or negative R");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) {
    set_error("fastfp_pack_simulate_residuals_blockn needs a plain-Fp pack (fastfp_pack_create_blockn without m_fix)");
    return FASTFP_ERR_INVALID;
  }
  if (!pk->ecorr) {
    set_error("fastfp_pack_simulate_residuals_blockn needs a block-diagonal N pack; a diagonal-N pack takes "
              "fastfp_pack_simulate_residuals");
    return FASTFP_ERR_INVALID;
  }
  const char* fn = "fastfp_pack_simulate_residuals_blockn";
  if (int rc = check_sim_args(pk, R, seed, first, phiinv, sig_freq, sig_amp, flags, fn)) return rc;
  if (int rc = check_res_limit(pk, R, fn)) return rc;
  for (int p = 0; p < pk->P && R > 0; ++p) {
    if (!slot_idx[p] || !slot_val[p] || !done_mask[p] || !toa_index[p] || !epoch[p] || !sqrt_j[p] || !beta[p]) {
      set_error(std::string(fn) + ": null per-pulsar array");
      return FASTFP_ERR_INVALID;
    }
    KernelCfg kc{};
    if (!sweep_config(sweep_rows(pk->meta[p].m, R, true), &kc) || n[p] < 1 || n[p] > 0x7fffff00LL ||
        n[p] % kc.ci != 0) {
      set_error(std::string(fn) + ": pulsar " + std::to_string(p) + ": the TOA count " + std::to_string(n[p]) +
                " of the residual layout must be a positive multiple of its chunk size " + std::to_string(kc.ci) +
                " (fastfp_sweep_chunk_toas(roundup8(m) + roundup8(R), 1))");
      return FASTFP_ERR_INVALID;
    }
  }
  const SimHost sim{seed, first, !(flags & FASTFP_SIM_NO_NOISE), phiinv, sig_freq, sig_amp,
                    toa_index, epoch, sqrt_j, beta};
  return replace_res(pk, R, {n, nullptr, nullptr, slot_idx, slot_val, done_mask}, stream, &sim);
}

int fastfp_fp_sweep_residuals(const fastfp_pack_t* pk, const double* freqs, int64_t F, double* out, int flags,
                              void* stream) {
  if (!pk || F < 0 || (F > 0 && (!freqs || !out))) {
    set_error("fastfp_fp_sweep_residuals: null argument or negative F");
    return FASTFP_ERR_INVALID;
  }
  if (pk->res.R == 0) {
    set_error("fastfp_fp_sweep_residuals: no residual realisations set (fastfp_pack_set_residuals)");
    return FASTFP_ERR_INVALID;
  }
  if (F == 0) return FASTFP_OK;
  const int P = pk->P;
  const int64_t R = pk->res.R;
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_out;
  if (int rc = c.stage(freqs, F, out, R * F, flags, &d_freqs, &d_out, &pk->out)) return rc;
  const int64_t FB = freq_batch(F, R * P);
  if (int rc = pk->res.terms.grow(R * P * std::min(FB, F))) return rc;
  for (int64_t lo = 0; lo < F; lo += FB) {
    const int64_t fb = std::min(FB, F - lo);
    const ResOut ro{pk->res.terms.get(), nullptr, nullptr, (int)R, P};
    if (int rc = launch_fp_sweep_res(pk, d_freqs + lo, fb, ro, c.st)) return rc;
    if (int rc = launch_reduce_terms_rows(pk->res.terms.get(), (int)R, P, fb, d_out + lo, F, c.st)) return rc;
  }
  return c.finish(flags, R * F, out, d_out, false);
}

// Fe-statistic sky scan: one sweep for the inner products of every (pulsar, frequency), then the combine kernel
int fastfp_fe_sweep(const fastfp_pack_t* pk, const double* freqs, int64_t F, const double* fplus, const double* fcross,
                    int64_t S, double* out, int flags, void* stream) {
  if (!pk || F < 0 || S < 0 || ((F > 0 && S > 0) && (!freqs || !fplus || !fcross || !out))) {
    set_error("fastfp_fe_sweep: null argument or negative size");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) { set_error("fastfp_fe_sweep needs a plain-Fp pack (fastfp_pack_create)"); return FASTFP_ERR_INVALID; }
  if (F == 0 || S == 0) return FASTFP_OK;
  const int P = pk->P;
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_out;
  if (int rc = c.stage(freqs, F, out, S * F, flags, &d_freqs, &d_out, &pk->out)) return rc;
  const int64_t FB = freq_batch(F, 5 * (int64_t)P + pk->rg_doubles_per_freq());
  // scratch: the inner products of one frequency batch, then the antenna patterns of the S sky positions
  ScratchLayout lay;
  const int64_t o_inner = lay.take(5 * (int64_t)P * std::min(FB, F)), o_fp = lay.take(S * P), o_fx = lay.take(S * P);
  if (int rc = pk->inner.grow(lay.total)) return rc;
  double* base = pk->inner.get();
  double *d_inner = base + o_inner, *d_fp = base + o_fp, *d_fx = base + o_fx;
  if (int rc = c.upload_sky(fplus, fcross, S * P, d_fp, d_fx)) return rc;
  for (int64_t lo = 0; lo < F; lo += FB) {
    const int64_t fb = std::min(FB, F - lo);
    if (int rc = launch_sweep(pk, d_freqs + lo, fb, FpOut{nullptr, d_inner}, c.st)) return rc;
    if (int rc = launch_fe_combine(d_inner, P, fb, d_fp, d_fx, S, d_out + lo, F, c.st)) return rc;
  }
  return c.finish(flags, S * F, out, d_out, true);
}

// Sky-maximised Fe: the same sweep per frequency batch, then a combine that reduces over the sky as it goes
int fastfp_fe_skymax(const fastfp_pack_t* pk, const double* freqs, int64_t F, const double* fplus, const double* fcross,
                     int64_t S, double* fe_max, int64_t* sky_index, int flags, void* stream) {
  if (!pk || F < 0 || S < 0 || (F > 0 && (!freqs || !fe_max || !sky_index || (S > 0 && (!fplus || !fcross))))) {
    set_error("fastfp_fe_skymax: null argument or negative size");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) { set_error("fastfp_fe_skymax needs a plain-Fp pack (fastfp_pack_create)"); return FASTFP_ERR_INVALID; }
  if (F == 0) return FASTFP_OK;
  if (S == 0) { set_error("fastfp_fe_skymax needs at least one sky position"); return FASTFP_ERR_INVALID; }
  const int P = pk->P;
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_max;
  if (int rc = c.stage(freqs, F, fe_max, F, flags, &d_freqs, &d_max, &pk->out)) return rc;
  const int64_t FB = freq_batch(F, 5 * (int64_t)P + pk->rg_doubles_per_freq());
  const int64_t fb0 = std::min(FB, F);
  const FeSkyPlan plan = fe_skymax_plan(fb0, S, pk->num_sms);
  // scratch, all in the pack's Fe buffer: the inner products of one frequency batch, the antenna patterns and the
  // weights of the S sky positions, the per-chunk bests of a split sky, and the indices on their way to host memory
  // (int64, 8 bytes per slot like the doubles). Like every scratch buffer of the pack it grows on demand and is kept
  // until the pack is destroyed: 5 P F_batch + 7 S P doubles, plus F for host outputs and a small split scratch; about
  // 750 MB after a call with S = 196 608 and P = 68. Allocating it per call instead costs a device allocation and
  // release per call, measured at up to several times the whole call at C2 sizes.
  const int64_t n_part = plan.nchunk > 1 ? plan.nchunk * fb0 : 0;
  const bool idx_to_host = !(flags & FASTFP_OUT_ON_DEVICE);
  ScratchLayout lay;
  const int64_t o_inner = lay.take(5 * (int64_t)P * fb0), o_fp = lay.take(S * P), o_fx = lay.take(S * P),
                o_w = lay.take(5 * S * P), o_part_v = lay.take(n_part), o_part_i = lay.take(n_part),
                o_idx = lay.take(idx_to_host ? F : 0);
  if (int rc = pk->inner.grow(lay.total)) return rc;
  double* base = pk->inner.get();
  double *d_inner = base + o_inner, *d_fp = base + o_fp, *d_fx = base + o_fx, *d_w = base + o_w;
  double* part_v = base + o_part_v;
  int64_t* part_i = reinterpret_cast<int64_t*>(base + o_part_i);
  int64_t* d_idx = idx_to_host ? reinterpret_cast<int64_t*>(base + o_idx) : sky_index;
  if (int rc = c.upload_sky(fplus, fcross, S * P, d_fp, d_fx)) return rc;
  if (int rc = launch_fe_sky_weights(d_fp, d_fx, S * P, d_w, c.st)) return rc;
  for (int64_t lo = 0; lo < F; lo += FB) {
    const int64_t fb = std::min(FB, F - lo);
    if (int rc = launch_sweep(pk, d_freqs + lo, fb, FpOut{nullptr, d_inner}, c.st)) return rc;
    if (int rc = launch_fe_skymax(d_inner, P, fb, d_w, S, plan, part_v, part_i, d_max + lo, d_idx + lo, c.st))
      return rc;
  }
  return c.finish(flags, F, fe_max, d_max, true, sky_index, d_idx);
}

// Sky-maximised Fe of each residual realisation (DESIGN.md section 5e): per frequency batch, the residual sweep writes
// the inner products and fe_skymax_res_kernel reduces over the sky
int fastfp_fe_skymax_residuals(const fastfp_pack_t* pk, const double* freqs, int64_t F, const double* fplus,
                               const double* fcross, int64_t S, double* fe_max, int64_t* sky_index, int flags,
                               void* stream) {
  if (!pk || F < 0 || S < 0 || (F > 0 && (!freqs || !fe_max || !sky_index || (S > 0 && (!fplus || !fcross))))) {
    set_error("fastfp_fe_skymax_residuals: null argument or negative size");
    return FASTFP_ERR_INVALID;
  }
  if (pk->nmfp) {
    set_error("fastfp_fe_skymax_residuals needs a plain-Fp pack (fastfp_pack_create)");
    return FASTFP_ERR_INVALID;
  }
  if (pk->res.R == 0) {
    set_error("fastfp_fe_skymax_residuals: no residual realisations set (fastfp_pack_set_residuals)");
    return FASTFP_ERR_INVALID;
  }
  if (F == 0) return FASTFP_OK;
  if (S == 0) { set_error("fastfp_fe_skymax_residuals needs at least one sky position"); return FASTFP_ERR_INVALID; }
  const int P = pk->P;
  const int64_t R = pk->res.R;
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_max;
  if (int rc = c.stage(freqs, F, fe_max, R * F, flags, &d_freqs, &d_max, &pk->out)) return rc;
  const int64_t FB = freq_batch(F, (2 * R + 3) * P);
  const int64_t fb0 = std::min(FB, F);
  // the sky is split across CTAs only in a single-batch call: the per-chunk bests are merged into (R, F) columns
  const FeSkyPlan plan = fe_skymax_res_plan(fb0, R, S, pk->num_sms, F <= FB);
  // scratch: (s|r_k), (c|r_k) of one frequency batch in the residual terms buffer; in the Fe buffer (s|s), (s|c), (c|c)
  // of the batch, the antenna patterns, the per-chunk bests of a split sky and the indices on their way to host memory
  const int64_t n_part = plan.nchunk > 1 ? plan.nchunk * R * fb0 : 0;
  const bool idx_to_host = !(flags & FASTFP_OUT_ON_DEVICE);
  if (int rc = pk->res.terms.grow(2 * R * P * fb0)) return rc;
  ScratchLayout lay;
  const int64_t o_mi = lay.take(3 * (int64_t)P * fb0), o_fp = lay.take(S * P), o_fx = lay.take(S * P),
                o_part_v = lay.take(n_part), o_part_i = lay.take(n_part), o_idx = lay.take(idx_to_host ? R * F : 0);
  if (int rc = pk->inner.grow(lay.total)) return rc;
  double* base = pk->inner.get();
  double *d_mi = base + o_mi, *d_fp = base + o_fp, *d_fx = base + o_fx, *part_v = base + o_part_v;
  int64_t* part_i = reinterpret_cast<int64_t*>(base + o_part_i);
  int64_t* d_idx = idx_to_host ? reinterpret_cast<int64_t*>(base + o_idx) : sky_index;
  if (int rc = c.upload_sky(fplus, fcross, S * P, d_fp, d_fx)) return rc;
  for (int64_t lo = 0; lo < F; lo += FB) {
    const int64_t fb = std::min(FB, F - lo);
    const ResOut ro{nullptr, pk->res.terms.get(), d_mi, (int)R, P};
    if (int rc = launch_fp_sweep_res(pk, d_freqs + lo, fb, ro, c.st)) return rc;
    if (int rc = launch_fe_skymax_res(pk->res.terms.get(), d_mi, P, R, fb, d_fp, d_fx, S, plan, part_v, part_i,
                                      d_max + lo, d_idx + lo, F, c.st))
      return rc;
  }
  return c.finish(flags, R * F, fe_max, d_max, true, sky_index, d_idx);
}

int fastfp_nmfp_sweep(const fastfp_pack_t* pk, const double* freqs, int64_t F,
                      const double* phiinv_var, int64_t D, double* out, int flags, void* stream) {
  if (!pk || F < 0 || D < 0 || ((F > 0 && D > 0) && (!freqs || !phiinv_var || !out))) {
    set_error("fastfp_nmfp_sweep: null argument or negative size");
    return FASTFP_ERR_INVALID;
  }
  if (!pk->nmfp) { set_error("this pack was built for plain Fp; use fastfp_fp_sweep"); return FASTFP_ERR_INVALID; }
  if (F == 0 || D == 0) return FASTFP_OK;
  PackCall c(pk, stream);
  const double* d_freqs;
  double* d_out;
  if (int rc = c.stage(freqs, F, out, D * F, flags, &d_freqs, &d_out, &pk->out)) return rc;
  const double* d_phi = phiinv_var;
  DeviceBuf<double> d_phi_tmp;
  if (!(flags & FASTFP_PARAMS_ON_DEVICE)) {
    FFP_CUDA(dev_alloc(&d_phi_tmp, (size_t)D * pk->mvar_total));
    FFP_CUDA(cudaMemcpyAsync(d_phi_tmp.get(), phiinv_var, (size_t)D * pk->mvar_total * 8,
                             cudaMemcpyHostToDevice, c.st));
    d_phi = d_phi_tmp.get();
  }
  int rc = nmfp_sweep_impl(pk, d_freqs, F, d_phi, D, d_out, c.st);
  if (!rc) rc = c.finish(flags, D * F, out, d_out, false);
  if (d_phi_tmp) cudaStreamSynchronize(c.st);  // the sweep reads the staged parameters until it ends
  return rc;
}

int fastfp_nmfp_tile_sizes(const fastfp_pack_t* pk, int64_t* z_per_tile, int64_t* a_per_tile) {
  if (!pk || !pk->nmfp || !z_per_tile || !a_per_tile) { set_error("fastfp_nmfp_tile_sizes: not an nmfp pack"); return FASTFP_ERR_INVALID; }
  *z_per_tile = (int64_t)pk->P * pk->mvpad * 64;
  *a_per_tile = (int64_t)pk->P * 160;
  return FASTFP_OK;
}

int fastfp_nmfp_stage_a(const fastfp_pack_t* pk, const double* freqs_dev, int64_t F, double* z_dev, double* a_dev,
                        void* stream) {
  if (!pk || !pk->nmfp || F <= 0 || !freqs_dev || !z_dev || !a_dev) {
    set_error("fastfp_nmfp_stage_a: not an nmfp pack, null argument or F <= 0");
    return FASTFP_ERR_INVALID;
  }
  PackCall c(pk, stream);
  if (int rc = c.select()) return rc;
  return nmfp_stage_a_impl(pk, freqs_dev, F, z_dev, a_dev, c.st);
}

int fastfp_nmfp_stage_b(const fastfp_pack_t* pk, const double* freqs_dev, int64_t F, const double* z_dev,
                        const double* a_dev, int64_t tiles_per_block, const double* phiinv_var_dev, int64_t D,
                        double* out_dev, void* stream) {
  if (!pk || !pk->nmfp || F <= 0 || D < 0 || tiles_per_block <= 0 || !freqs_dev || !z_dev || !a_dev ||
      (D > 0 && (!phiinv_var_dev || !out_dev))) {
    set_error("fastfp_nmfp_stage_b: not an nmfp pack, null argument or bad size");
    return FASTFP_ERR_INVALID;
  }
  if (D == 0) return FASTFP_OK;
  PackCall c(pk, stream);
  if (int rc = c.select()) return rc;
  return nmfp_stage_b_only(pk, freqs_dev, F, z_dev, a_dev, (int)tiles_per_block, phiinv_var_dev, D, out_dev, c.st);
}

int fastfp_nmfp_stage_timing(fastfp_pack_t* pk, int enable) {
  if (!pk || !pk->nmfp) { set_error("fastfp_nmfp_stage_timing: not an nmfp pack"); return FASTFP_ERR_INVALID; }
  pk->time_stages = enable != 0;
  return FASTFP_OK;
}

int fastfp_nmfp_stage_ms(const fastfp_pack_t* pk, double* ms3) {
  if (!pk || !pk->nmfp || !ms3) { set_error("fastfp_nmfp_stage_ms: not an nmfp pack"); return FASTFP_ERR_INVALID; }
  for (int i = 0; i < 3; ++i) ms3[i] = pk->stage_ms[i];
  return FASTFP_OK;
}

int fastfp_powerlaw_phiinv(const fastfp_pack_t* pk, const double* const* Ffreqs,
                           const double* log10_A, const double* gamma, int64_t D,
                           const double* curn_Ffreqs, int64_t ncurn, const double* curn_log10_A,
                           const double* curn_gamma, double* phiinv_var_dev, void* stream) {
  if (!pk || !pk->nmfp || !Ffreqs || !log10_A || !gamma || D < 0 || !phiinv_var_dev ||
      (ncurn > 0 && (!curn_Ffreqs || !curn_log10_A || !curn_gamma))) {
    set_error("fastfp_powerlaw_phiinv: invalid argument");
    return FASTFP_ERR_INVALID;
  }
  if (D == 0) return FASTFP_OK;
  PackCall c(pk, stream);
  if (int rc = c.select()) return rc;
  return powerlaw_phiinv_impl(pk, Ffreqs, log10_A, gamma, D, curn_Ffreqs, ncurn, curn_log10_A,
                              curn_gamma, phiinv_var_dev, c.st);
}

static int xcy_run(int device, int64_t n, int64_t m, const double* Nvec, const double* T, const double* sigma,
                   const double* x, const double* y, const double* x0, double* out, void* stream) {
  if (n < 1 || m < 1 || !Nvec || !T || !sigma || !x || !y || !out) {
    set_error("fastfp_xcy: null argument or non-positive size");
    return FASTFP_ERR_INVALID;
  }
  DeviceGuard g(device);
  if (!g.ok) { set_error("cannot select CUDA device " + std::to_string(device)); return FASTFP_ERR_CUDA; }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t tot = (size_t)(4 * n + n * m + m * m) + (size_t)(m * m + 3 * m + 2);
  DeviceBuf<double> d;
  FFP_CUDA(dev_alloc(&d, tot));
  double *dN = d.get(), *dx = dN + n, *dy = dx + n, *dx0 = dy + n, *dT = dx0 + n, *dS = dT + n * m, *dW = dS + m * m;
  double* dO = dW + (m * m + 3 * m);
  cudaError_t e = cudaMemcpyAsync(dN, Nvec, n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dx, x, n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dy, y, n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && x0) e = cudaMemcpyAsync(dx0, x0, n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dT, T, n * m * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dS, sigma, m * m * 8, cudaMemcpyHostToDevice, st);
  int rc = 0;
  if (e != cudaSuccess) rc = cuda_fail(e, "fastfp_xcy upload");
  if (!rc) rc = launch_xcy(n, m, dN, dT, dS, dx, dy, x0 ? dx0 : nullptr, dW, dO, st);
  if (!rc) {
    e = cudaMemcpyAsync(out, dO, 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = cuda_fail(e, "fastfp_xcy download");
  }
  return rc;
}

int fastfp_xcy(int device, int64_t n, int64_t m, const double* Nvec, const double* T,
               const double* sigma, const double* x, const double* y, double* out, void* stream) {
  return xcy_run(device, n, m, Nvec, T, sigma, x, y, nullptr, out, stream);
}

int fastfp_xcy_blockn(int device, int64_t n, int64_t m, const double* Nvec, const double* T,
                      const double* sigma, const double* x, const double* xw, const double* yw,
                      double* out, void* stream) {
  if (!xw || !yw) { set_error("fastfp_xcy_blockn: null argument"); return FASTFP_ERR_INVALID; }
  return xcy_run(device, n, m, Nvec, T, sigma, xw, yw, x, out, stream);
}

int fastfp_tnt(int device, int64_t n, int64_t m, const double* Nvec, const double* T, const double* phiinv,
               double* out, void* stream) {
  if (n < 1 || m < 1 || !Nvec || !T || !out) {
    set_error("fastfp_tnt: null argument or non-positive size");
    return FASTFP_ERR_INVALID;
  }
  DeviceGuard g(device);
  if (!g.ok) { set_error("cannot select CUDA device " + std::to_string(device)); return FASTFP_ERR_CUDA; }
  cudaStream_t st = (cudaStream_t)stream;
  const int nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(64, n / 256));
  const size_t tot = (size_t)(n + n * m + m + m * m) + (size_t)nsplit * m * m;
  DeviceBuf<double> d;
  FFP_CUDA(dev_alloc(&d, tot));
  double *dN = d.get(), *dT = dN + n, *dP = dT + n * m, *dO = dP + m, *dW = dO + m * m;
  cudaError_t e = cudaMemcpyAsync(dN, Nvec, n * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dT, T, n * m * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && phiinv) e = cudaMemcpyAsync(dP, phiinv, m * 8, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(dW, 0, (size_t)nsplit * m * m * 8, st);
  int rc = 0;
  if (e != cudaSuccess) rc = cuda_fail(e, "fastfp_tnt upload");
  if (!rc) rc = launch_tnt(n, m, dN, dT, phiinv ? dP : nullptr, dW, nsplit, dO, st);
  if (!rc) {
    e = cudaMemcpyAsync(out, dO, m * m * 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) rc = cuda_fail(e, "fastfp_tnt download");
  }
  return rc;
}

int fastfp_fp64_peak(int device, int kind, int iters, double* tflops, double* ms) {
  if (!tflops || !ms || iters < 1 || kind < 0 || kind > 25) {
    set_error("fastfp_fp64_peak: invalid argument");
    return FASTFP_ERR_INVALID;
  }
  DeviceGuard g(device);
  if (!g.ok) { set_error("cannot select CUDA device"); return FASTFP_ERR_CUDA; }
  if (kind == 17 || kind == 18) return run_i8_peak(kind, iters, tflops, ms);
  return run_fp64_peak(kind, iters, tflops, ms);
}

}  // extern "C"
