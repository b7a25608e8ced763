// Residual batches drawn on the device (DESIGN.md section 5g). A realisation r = n + T Phi^(1/2) zeta of the noise
// model (n: white noise, plus the ECORR epoch draws of a block-diagonal N, plus an optional Earth-term signal) enters
// the sweep only through w = C^-1 r, and by Woodbury (C^-1 T Phi = N^-1 T Sigma^-1)
//   w = N^-1 n - G^T (G n - L^-1 (sqrt(phiinv) o zeta)),      G = L^-1 T^T N^-1,  Sigma = L L^T
// so the pack's G and L are all it needs: sim_noise_kernel writes n where the host staging of a residual batch would
// be, ur_batch_kernel forms U = G n, sim_basis_kernel subtracts L^-1 (sqrt(phiinv) o zeta) from U, and w_batch_kernel
// finishes w as for uploaded realisations.
//
// Random stream (normative, include/fastfp_b200.h): Philox4x64-10 with key (seed, 0) and counter (q, k, p, tag), k the
// global realisation index, p the pulsar, tag 0 white noise (by original TOA index), 1 ECORR (by epoch), 2 basis
// columns; block q gives normals 4q .. 4q+3 by Box-Muller of the uniforms ((x >> 11) + 0.5) 2^-53.
#include <algorithm>
#include <cmath>

#include "ffp_internal.cuh"
#include "ffp_sincos.cuh"

namespace ffp {

namespace {

constexpr uint64_t kPhiloxM0 = 0xD2E7470EE14C6C93ULL, kPhiloxM1 = 0xCA5A826395121157ULL;
constexpr uint64_t kPhiloxW0 = 0x9E3779B97F4A7C15ULL, kPhiloxW1 = 0xBB67AE8584CAA73BULL;

// normal number j of stream (seed, k, p, tag)
__device__ double sim_normal(uint64_t seed, uint64_t k, uint64_t p, uint64_t tag, int64_t j) {
  uint64_t c0 = (uint64_t)j >> 2, c1 = k, c2 = p, c3 = tag, k0 = seed, k1 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t hi0 = __umul64hi(kPhiloxM0, c0), lo0 = kPhiloxM0 * c0;
    const uint64_t hi1 = __umul64hi(kPhiloxM1, c2), lo1 = kPhiloxM1 * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += kPhiloxW0;
    k1 += kPhiloxW1;
  }
  const bool second = (j & 2) != 0;  // pair (u2, u3) gives normals 4q+2, 4q+3
  const uint64_t a = second ? c2 : c0, b = second ? c3 : c1;
  const double u0 = ((double)(a >> 11) + 0.5) * 0x1p-53, u1 = ((double)(b >> 11) + 0.5) * 0x1p-53;
  double s, c;
  sincos(6.283185307179586 * u1, &s, &c);
  return sqrt(-2.0 * log(u0)) * ((j & 1) ? s : c);
}

// t and 1/N of TOA position i of pulsar pm in the pack's packets
__device__ __forceinline__ const double* toa_at(const double* packets, const PulsarMeta& pm, int i) {
  return packets + pm.pk_off + (size_t)(i / pm.ci) * (pm.ci * (4 + pm.mpad)) + 4 * (i % pm.ci);
}

}  // namespace

// One thread per (segment, realisation, pulsar): with a diagonal N a segment is one TOA position; with a block N it is
// an epoch's run of positions (or one position outside any epoch), so the thread that draws the epoch also forms its
// Sherman-Morrison sum A_e = sum_i n_i / N_i, in position order, and writes res_w = n - beta_e A_e (the (N^-1 n) * Nvec
// of blockn.solve_rows). Writes n (and res_w) into the (R, n_shared) staging blocks at R * smeta.raw_off.
__global__ void __launch_bounds__(128) sim_noise_kernel(double* __restrict__ res, double* __restrict__ res_w,
                                                        const PulsarMeta* __restrict__ smeta,
                                                        const PulsarMeta* __restrict__ meta,
                                                        const double* __restrict__ packets, int R, int P, SimArgs a) {
  const int p = blockIdx.z, k = blockIdx.y;
  const PulsarMeta sm = smeta[p], pm = meta[p];
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  const bool blockn = a.seg != nullptr;
  const int units = blockn ? (int)(a.seg_off[p + 1] - a.seg_off[p] - 1) : sm.n;
  if (u >= units) return;
  const int lo = blockn ? a.seg[a.seg_off[p] + u] : u, hi = blockn ? a.seg[a.seg_off[p] + u + 1] : u + 1;
  const int e = blockn ? a.seg_epoch[a.seg_off[p] + u] : -1;
  const uint64_t kg = a.first + (uint64_t)k;
  // Earth-term signal: the sweep's phase ((2 pi) f) t, each product rounded once, and its sincos range rule
  double As = 0.0, Ac = 0.0, omega = 0.0;
  bool fast = true;
  const bool sig = a.sig_freq != nullptr;
  if (sig) {
    omega = __dmul_rn(6.283185307179586, a.sig_freq[k]);
    As = a.sig_amp[((size_t)k * P + p) * 2];
    Ac = a.sig_amp[((size_t)k * P + p) * 2 + 1];
    fast = fabs(omega) * pm.tabs_max <= 0.999 * FFP_SINCOS_MAX;
  }
  const double xe = a.noise && e >= 0 ? a.sqrt_j[a.ep_off[p] + e] * sim_normal(a.seed, kg, p, 1, e) : 0.0;
  double* rp = res + (size_t)R * sm.raw_off + (size_t)k * sm.n;
  double A = 0.0;
  for (int i = lo; i < hi; ++i) {
    const double* tv = toa_at(packets, pm, i);
    const double ninv = tv[1];
    const int o = blockn ? a.toa_index[sm.raw_off + i] : i;
    double x = 0.0;
    if (o >= 0) {
      if (a.noise) x = fma(sqrt(1.0 / ninv), sim_normal(a.seed, kg, p, 0, o), xe);
      if (sig) {
        const double ph = __dmul_rn(omega, tv[0]);
        double s, c;
        if (fast) sincos_cw(ph, &s, &c);
        else sincos(ph, &s, &c);
        x += fma(As, s, Ac * c);
      }
    }
    rp[i] = x;
    A = fma(x, ninv, A);
  }
  if (!res_w) return;
  double* wp = res_w + (size_t)R * sm.raw_off + (size_t)k * sm.n;
  const double bA = e >= 0 ? a.beta[a.ep_off[p] + e] * A : 0.0;
  for (int i = lo; i < hi; ++i) wp[i] = rp[i] - bA;
}

// One warp per (realisation, pulsar): U[p][k] -= L^-1 (sqrt(phiinv) o zeta) by column-oriented forward substitution on
// the pack's factor (row-major m x m at L_off, lower part). Each entry of v is updated by the same sequence of FMAs
// whichever lane holds it, so the result does not depend on where the realisation sits in the batch.
__global__ void __launch_bounds__(256) sim_basis_kernel(double* __restrict__ U, int ld, const double* __restrict__ Lbuf,
                                                        const PulsarMeta* __restrict__ meta, int R, SimArgs a) {
  __shared__ double vs[8][MAX_M];
  const int lane = threadIdx.x & 31, wq = threadIdx.x >> 5;
  const int p = blockIdx.y, k = blockIdx.x * 8 + wq;
  if (k >= R) return;  // warp-uniform; the warps do not synchronise with each other
  const PulsarMeta pm = meta[p];
  const int m = pm.m;
  const double* L = Lbuf + pm.L_off;
  double* v = vs[wq];
  const uint64_t kg = a.first + (uint64_t)k;
  for (int j = lane; j < m; j += 32) v[j] = sqrt(a.phiinv[(size_t)p * MAX_M + j]) * sim_normal(a.seed, kg, p, 2, j);
  __syncwarp();
  double* Up = U + ((size_t)p * R + k) * ld;
  for (int j = 0; j < m; ++j) {
    const double y = v[j] / L[(size_t)j * m + j];
    for (int i = j + 1 + lane; i < m; i += 32) v[i] = fma(-L[(size_t)i * m + j], y, v[i]);
    if (lane == 0) Up[j] -= y;
    __syncwarp();
  }
}

// segments of one block-N pulsar over its n_shared staging positions: maximal runs of one epoch, every other position
// alone. FASTFP_ERR_INVALID if an epoch is split into several runs or out of range.
static int sim_segments(const int32_t* epoch, const int32_t* toa_index, int n, int p, std::vector<int>* seg,
                        std::vector<int>* seg_ep, int* nep) {
  for (int i = 0; i < n; ++i) {
    if (epoch[i] < -1 || epoch[i] >= n || toa_index[i] < -1 || (epoch[i] >= 0 && toa_index[i] < 0)) {
      set_error("simulated residual batch: pulsar " + std::to_string(p) + ": bad epoch or TOA index at position " +
                std::to_string(i));
      return FASTFP_ERR_INVALID;
    }
  }
  std::vector<char> seen;
  *nep = 0;
  for (int i = 0; i < n;) {
    const int e = epoch[i];
    int j = i + 1;
    if (e >= 0) {
      while (j < n && epoch[j] == e) ++j;
      if ((int)seen.size() <= e) seen.resize(e + 1, 0);
      if (seen[e]) {
        set_error("simulated residual batch: pulsar " + std::to_string(p) + ": epoch " + std::to_string(e) +
                  " is not one contiguous run of the layout");
        return FASTFP_ERR_INVALID;
      }
      seen[e] = 1;
      *nep = std::max(*nep, e + 1);
    }
    seg->push_back(i);
    seg_ep->push_back(e);
    i = j;
  }
  seg->push_back(n);
  seg_ep->push_back(-1);  // keeps seg_epoch aligned with seg
  return 0;
}

template <typename T>
static int upload(DeviceBuf<T>* buf, const T* src, size_t count, cudaStream_t st) {
  FFP_CUDA(dev_alloc(buf, std::max<size_t>(count, 1)));
  if (count) FFP_CUDA(cudaMemcpyAsync(buf->get(), src, count * sizeof(T), cudaMemcpyHostToDevice, st));
  return 0;
}

int launch_sim_noise(const SimHost& s, const fastfp_pack* pk, const std::vector<PulsarMeta>& smeta,
                     const PulsarMeta* d_smeta, int64_t R, double* d_res, double* d_res_w, SimStage* ss,
                     cudaStream_t st) {
  const int P = pk->P;
  SimArgs& a = ss->args;
  a = SimArgs{};
  a.seed = (uint64_t)s.seed;
  a.first = (uint64_t)s.first;
  a.noise = s.noise ? 1 : 0;
  std::vector<double> phi((size_t)P * MAX_M, 0.0);
  for (int p = 0; p < P; ++p) std::copy(s.phiinv[p], s.phiinv[p] + pk->meta[p].m, phi.begin() + (size_t)p * MAX_M);
  // the host vectors must outlive the asynchronous copies: ss keeps them until the batch is built
  ss->host_phi = std::move(phi);
  if (int rc = upload(&ss->phiinv, ss->host_phi.data(), ss->host_phi.size(), st)) return rc;
  a.phiinv = ss->phiinv.get();
  if (s.sig_freq) {
    if (int rc = upload(&ss->sig_freq, s.sig_freq, (size_t)R, st)) return rc;
    if (int rc = upload(&ss->sig_amp, s.sig_amp, (size_t)R * P * 2, st)) return rc;
    a.sig_freq = ss->sig_freq.get();
    a.sig_amp = ss->sig_amp.get();
  }
  int units = 0;
  if (s.toa_index) {
    std::vector<int>& idx = ss->host_idx;
    std::vector<int>& seg = ss->host_seg;
    std::vector<int>& sep = ss->host_seg_ep;
    std::vector<int64_t>& soff = ss->host_seg_off;
    std::vector<int64_t>& eoff = ss->host_ep_off;
    std::vector<double>& sj = ss->host_sqrt_j;
    std::vector<double>& be = ss->host_beta;
    soff.assign(1, 0);
    eoff.assign(1, 0);
    for (int p = 0; p < P; ++p) {
      const PulsarMeta& sm = smeta[p];
      int nep = 0;
      const size_t before = seg.size();
      if (int rc = sim_segments(s.epoch[p], s.toa_index[p], sm.n, p, &seg, &sep, &nep)) return rc;
      units = std::max(units, (int)(seg.size() - before) - 1);
      soff.push_back((int64_t)seg.size());
      idx.insert(idx.end(), s.toa_index[p], s.toa_index[p] + sm.n);
      for (int e = 0; e < nep; ++e) {
        if (!(s.sqrt_j[p][e] >= 0.0) || !std::isfinite(s.sqrt_j[p][e]) || !std::isfinite(s.beta[p][e])) {
          set_error("simulated residual batch: pulsar " + std::to_string(p) + ": sqrt_j and beta of epoch " +
                    std::to_string(e) + " must be finite, sqrt_j >= 0");
          return FASTFP_ERR_INVALID;
        }
      }
      sj.insert(sj.end(), s.sqrt_j[p], s.sqrt_j[p] + nep);
      be.insert(be.end(), s.beta[p], s.beta[p] + nep);
      eoff.push_back((int64_t)sj.size());
    }
    if (int rc = upload(&ss->toa_index, idx.data(), idx.size(), st)) return rc;
    if (int rc = upload(&ss->seg, seg.data(), seg.size(), st)) return rc;
    if (int rc = upload(&ss->seg_epoch, sep.data(), sep.size(), st)) return rc;
    if (int rc = upload(&ss->seg_off, soff.data(), soff.size(), st)) return rc;
    if (int rc = upload(&ss->ep_off, eoff.data(), eoff.size(), st)) return rc;
    if (int rc = upload(&ss->sqrt_j, sj.data(), sj.size(), st)) return rc;
    if (int rc = upload(&ss->beta, be.data(), be.size(), st)) return rc;
    a.toa_index = ss->toa_index.get();
    a.seg = ss->seg.get();
    a.seg_epoch = ss->seg_epoch.get();
    a.seg_off = ss->seg_off.get();
    a.ep_off = ss->ep_off.get();
    a.sqrt_j = ss->sqrt_j.get();
    a.beta = ss->beta.get();
  } else {
    for (auto& sm : smeta) units = std::max(units, sm.n);
  }
  sim_noise_kernel<<<dim3((units + 127) / 128, (unsigned)R, P), 128, 0, st>>>(d_res, d_res_w, d_smeta, pk->core.meta.get(),
                                                                             pk->core.packets.get(), (int)R, P, a);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

int launch_sim_basis(const fastfp_pack* pk, int64_t R, double* d_U, int ld, const SimStage& ss, cudaStream_t st) {
  sim_basis_kernel<<<dim3((unsigned)((R + 7) / 8), pk->P), 256, 0, st>>>(d_U, ld, pk->core.L.get(), pk->core.meta.get(),
                                                                       (int)R, ss.args);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ffp
