// One-time, frequency-independent per-pulsar work for the plain-Fp path (DESIGN.md section 3):
//   Sigma = L L^T,  G = L^-1 T^T N^-1  (m x n),  u_r = G r,  w = C^-1 r = N^-1 r - G^T u_r
// and the packed, tile-contiguous layout the sweep kernel streams with one TMA bulk copy per
// chunk: packet = [ (t, 1/N, w, 0)[CI] | G in mma-fragment order (g_frag_index) ]  (CI = 16 or 32).
//
// The reference recomputes all of this for every frequency: T^T N^-1 x twice per get_xCy
// (fastfp/utils.py:51-52) and an LU solve of Sigma per call (utils.py:54), six calls per
// (frequency, pulsar) (fastfp/fastfp.py:81-88). With Sigma = L L^T,
//   (x|y) = x^T N^-1 y - (G x).(G y)        and       (x|r) = x . w
// so the per-frequency work collapses to Y = G [s c] plus five weighted dot products.
#include "ffp_internal.cuh"

namespace ffp {

// In-place lower Cholesky of the m x m matrix at Lbuf + L_off (row-major; the strictly upper
// part is left untouched and never read), stopped after the first mfix columns. One CTA per
// pulsar. For a plain-Fp pack mfix = m (full factor). For an nmfp pack the leading mfix x mfix
// block becomes L_X, the lower-left block becomes Sigma_VX L_X^-T, and the trailing block is left
// holding the Schur complement TNT_VV - Sigma_VX Sigma_XX^-1 Sigma_XV (lower part).
// info[p] = j+1 if pivot j is not positive (the factor then carries NaN, which propagates like
// the reference's non-raising jnp.linalg.solve on a singular Sigma).
__global__ void chol_kernel(double* __restrict__ Lbuf, const PulsarMeta* __restrict__ meta,
                            int* __restrict__ info) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int m = pm.m;
  double* A = Lbuf + pm.L_off;
  __shared__ double djj;
  for (int j = 0; j < pm.mfix; ++j) {
    if (threadIdx.x == 0) {
      const double d = A[(size_t)j * m + j];
      if (!(d > 0.0) && info[blockIdx.x] == 0) info[blockIdx.x] = j + 1;
      djj = sqrt(d);
      A[(size_t)j * m + j] = djj;
    }
    __syncthreads();
    const double d = djj;
    for (int i = j + 1 + threadIdx.x; i < m; i += blockDim.x)
      A[(size_t)i * m + j] = A[(size_t)i * m + j] / d;
    __syncthreads();
    const int cnt = m - j - 1;
    for (int idx = threadIdx.x; idx < cnt * cnt; idx += blockDim.x) {
      const int ii = idx / cnt, kk = idx - ii * cnt;
      if (kk <= ii) {
        const int i = j + 1 + ii, k = j + 1 + kk;
        A[(size_t)i * m + k] =
            fma(-A[(size_t)i * m + j], A[(size_t)k * m + j], A[(size_t)i * m + k]);
      }
    }
    __syncthreads();
  }
}

// One thread per (padded) TOA: forward-substitute L g = T_i^T / N_i and scatter t, 1/N and g
// into the packet layout. Padded TOAs get zeros (weight 0: they add nothing to any sum).
__global__ void build_packets_kernel(double* __restrict__ packets,
                                     const PulsarMeta* __restrict__ meta,
                                     const double* __restrict__ Lbuf,
                                     const double* __restrict__ toas,
                                     const double* __restrict__ Nvec,
                                     const double* __restrict__ T,
                                     const int* __restrict__ slot_idx,
                                     const double* __restrict__ slot_val) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int CI = pm.ci;
  if (i >= pm.nch * CI) return;
  const int m = pm.m, mp = pm.mpad;
  const int pkw = CI * (4 + mp);
  double* pk = packets + pm.pk_off + (size_t)(i / CI) * pkw;
  const int il = i % CI;
  const bool valid = i < pm.n;
  const double ninv = valid ? 1.0 / Nvec[pm.raw_off + i] : 0.0;
  pk[4 * il] = valid ? toas[pm.raw_off + i] : 0.0;
  pk[4 * il + 1] = ninv;
  pk[4 * il + 2] = 0.0;  // w, filled by w_kernel
  pk[4 * il + 3] = 0.0;
  double* gp = pk + 4 * CI;  // G part, fragment order
  const int nmb = mp >> 3;
  if (!valid) {
    for (int j = 0; j < mp; ++j) gp[g_frag_index(il, j, nmb)] = 0.0;
    return;
  }
  const double* L = Lbuf + pm.L_off;
  const double* Ti = T + pm.T_off + (size_t)i * m;
  double g[MAX_M];  // thread-local column of G (local memory; one-time work)
  // rows below mfix: g = L_X^-1 T_X^T / N (forward substitution); rows of the per-draw block
  // (nmfp): g = T_V^T / N - (Sigma_VX L_X^-T) g_X, i.e. the same recurrence without the division
  const int mfix = pm.mfix;
  for (int j = 0; j < m; ++j) {
    double acc = Ti[j] * ninv;
    const double* Lj = L + (size_t)j * m;
    const int kend = j < mfix ? j : mfix;
    for (int k = 0; k < kend; ++k) acc = fma(-Lj[k], g[k], acc);
    g[j] = j < mfix ? acc / Lj[j] : acc;
    gp[g_frag_index(il, j, nmb)] = g[j];
  }
  for (int j = m; j < mp; ++j) gp[g_frag_index(il, j, nmb)] = 0.0;
  // block-diagonal N: the last row block holds the epoch slots; this TOA feeds sqrt(beta_e)/N_i
  // into the slot of its epoch (fp_sweep_kernel folds the slot sums when the epoch ends)
  if (slot_idx != nullptr) {
    const int sidx = slot_idx[pm.raw_off + i];
    if (sidx >= 0) gp[g_frag_index(il, mp - 8 + sidx, nmb)] = slot_val[pm.raw_off + i];
  }
}

// u_r[j] = sum_i G[j][i] r_i. One CTA per pulsar, one warp per basis row at a time; lanes
// stride over TOAs, fixed-order shuffle tree: deterministic.
__global__ void ur_kernel(const double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                          const double* __restrict__ res, double* __restrict__ ur) {
  const PulsarMeta pm = meta[blockIdx.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int CI = pm.ci;
  const int mp = pm.mpad, pkw = CI * (4 + mp);
  const double* pk0 = packets + pm.pk_off;
  for (int j = wid; j < pm.m; j += nw) {
    double acc = 0.0;
    for (int i = lane; i < pm.n; i += 32) {
      const double g = pk0[(size_t)(i / CI) * pkw + 4 * CI + g_frag_index(i % CI, j, mp >> 3)];
      acc = fma(g, res[pm.raw_off + i], acc);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) ur[(size_t)blockIdx.x * MAX_M + j] = acc;
  }
}

// w_i = r_i / N_i - sum_{j < mfix} G[j][i] u_r[j]   (= (C^-1 r)_i for a plain-Fp pack)
__global__ void w_kernel(double* __restrict__ packets, const PulsarMeta* __restrict__ meta,
                         const double* __restrict__ res, const double* __restrict__ ur) {
  const PulsarMeta pm = meta[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pm.n) return;
  const int CI = pm.ci;
  const int mp = pm.mpad, pkw = CI * (4 + mp);
  double* pk = packets + pm.pk_off + (size_t)(i / CI) * pkw;
  const int il = i % CI;
  const double* gp = pk + 4 * CI;
  const double* u = ur + (size_t)blockIdx.y * MAX_M;
  double acc = 0.0;
  for (int j = 0; j < pm.mfix; ++j) acc = fma(gp[g_frag_index(il, j, mp >> 3)], u[j], acc);
  pk[4 * il + 2] = res[pm.raw_off + i] * pk[4 * il + 1] - acc;
}

int launch_fp_precompute(fastfp_pack* pk, const double* d_toas, const double* d_res,
                         const double* d_Nvec, const double* d_T, cudaStream_t st, double* d_ur_keep,
                         const BlockNDev* bn) {
  const int P = pk->P;
  int nmax = 0;
  for (auto& m : pk->meta) nmax = m.nch * m.ci > nmax ? m.nch * m.ci : nmax;
  DeviceBuf<double> ur_tmp;
  double* d_ur = d_ur_keep;
  if (!d_ur) {
    FFP_CUDA(dev_alloc(&ur_tmp, (size_t)P * MAX_M));
    d_ur = ur_tmp.get();
  }
  chol_kernel<<<P, 256, 0, st>>>(pk->d_L, pk->d_meta, pk->d_info);
  dim3 g1((nmax + 127) / 128, P);
  build_packets_kernel<<<g1, 128, 0, st>>>(pk->d_packets, pk->d_meta, pk->d_L, d_toas, d_Nvec, d_T,
                                           bn ? bn->slot_idx : nullptr, bn ? bn->slot_val : nullptr);
  ur_kernel<<<P, 256, 0, st>>>(pk->d_packets, pk->d_meta, d_res, d_ur);
  // with a block-diagonal N the first term of w is N^-1 r, supplied as (N^-1 r) * Nvec
  w_kernel<<<g1, 128, 0, st>>>(pk->d_packets, pk->d_meta, bn ? bn->res_w : d_res, d_ur);
  g_launches += 4;
  FFP_CUDA(cudaGetLastError());
  FFP_CUDA(cudaStreamSynchronize(st));
  // the factorisation status comes back with the pack: a non-positive pivot means Sigma was not numerically
  // SPD; the factor then carries NaN, which propagates like the reference's non-raising solve -- but the
  // caller can ask which pulsar it was (fastfp_pack_factor_info; the Python mirror warns)
  pk->info.assign(P, 0);
  FFP_CUDA(cudaMemcpy(pk->info.data(), pk->d_info, sizeof(int) * P, cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace ffp
