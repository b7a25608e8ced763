// get_xCy on the device: x^T C^-1 y = x^T N^-1 y - (T^T N^-1 x)^T Sigma^-1 (T^T N^-1 y),
// operation for operation as the reference writes it (fastfp/utils.py:49-54), including a
// general LU solve with partial pivoting (what jnp.linalg.solve performs), so it also accepts
// a Sigma that is not positive definite. One CTA; this is the API-parity op, not the hot path.
// For a block-diagonal N the caller passes xw = (N^-1 x) * Nvec and yw likewise (Sherman-Morrison
// on the host): then xw / Nvec = N^-1 x, and x^T N^-1 y = sum x_i * (yw_i / Nvec_i) with the raw x.
#include "ffp_internal.cuh"

namespace ffp {

// work layout (doubles): LU[m*m] | TNx[m] | TNy[m] | sol[m] | xNy[1]. The threads exchange values through `work`
// across __syncthreads(), so it must not be __restrict__: that would let the compiler move its loads across the
// barriers.
__global__ void xcy_kernel(int64_t n, int m, const double* __restrict__ Nvec,
                           const double* __restrict__ T, const double* __restrict__ sigma,
                           const double* __restrict__ x, const double* __restrict__ y,
                           const double* __restrict__ x0, double* work, double* out) {
  double* LU = work;
  double* TNx = work + (size_t)m * m;
  double* TNy = TNx + m;
  double* sol = TNy + m;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  __shared__ double red[32];
  __shared__ int piv;

  // TNx = T^T (x / Nvec), TNy = T^T (y / Nvec): one warp per column, lanes stride TOAs
  for (int j = wid; j < m; j += nw) {
    double ax = 0.0, ay = 0.0;
    for (int64_t i = lane; i < n; i += 32) {
      const double t = T[i * m + j];
      ax = fma(t, x[i] / Nvec[i], ax);
      ay = fma(t, y[i] / Nvec[i], ay);
    }
    for (int o = 16; o > 0; o >>= 1) {
      ax += __shfl_xor_sync(0xffffffffu, ax, o);
      ay += __shfl_xor_sync(0xffffffffu, ay, o);
    }
    if (lane == 0) { TNx[j] = ax; TNy[j] = ay; }
  }
  // xNy = x . (y / Nvec)
  double a = 0.0;
  for (int64_t i = tid; i < n; i += blockDim.x) a = fma(x0[i], y[i] / Nvec[i], a);
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) red[wid] = a;
  for (int idx = tid; idx < m * m; idx += blockDim.x) LU[idx] = sigma[idx];
  __syncthreads();
  double xNy = 0.0;
  for (int w = 0; w < nw; ++w) xNy += red[w];
  for (int j = tid; j < m; j += blockDim.x) sol[j] = TNy[j];
  __syncthreads();

  // LU with partial pivoting, right-hand side carried along
  for (int k = 0; k < m; ++k) {
    if (tid == 0) {
      int best = k;
      double bv = fabs(LU[(size_t)k * m + k]);
      for (int i = k + 1; i < m; ++i) {
        const double v = fabs(LU[(size_t)i * m + k]);
        if (v > bv) { bv = v; best = i; }
      }
      piv = best;
    }
    __syncthreads();
    const int pr = piv;
    if (pr != k) {
      for (int j = tid; j < m; j += blockDim.x) {
        const double t0 = LU[(size_t)k * m + j];
        LU[(size_t)k * m + j] = LU[(size_t)pr * m + j];
        LU[(size_t)pr * m + j] = t0;
      }
      if (tid == 0) { const double t0 = sol[k]; sol[k] = sol[pr]; sol[pr] = t0; }
    }
    __syncthreads();
    const double d = LU[(size_t)k * m + k];
    for (int i = k + 1 + tid; i < m; i += blockDim.x) LU[(size_t)i * m + k] = LU[(size_t)i * m + k] / d;
    __syncthreads();
    const int cnt = m - k - 1;
    for (int idx = tid; idx < cnt * cnt; idx += blockDim.x) {
      const int i = k + 1 + idx / cnt, j = k + 1 + idx % cnt;
      LU[(size_t)i * m + j] = fma(-LU[(size_t)i * m + k], LU[(size_t)k * m + j], LU[(size_t)i * m + j]);
    }
    for (int i = k + 1 + tid; i < m; i += blockDim.x) sol[i] = fma(-LU[(size_t)i * m + k], sol[k], sol[i]);
    __syncthreads();
  }
  // back substitution (serial in k, parallel over rows above)
  for (int k = m - 1; k >= 0; --k) {
    if (tid == 0) sol[k] = sol[k] / LU[(size_t)k * m + k];
    __syncthreads();
    const double sk = sol[k];
    for (int i = tid; i < k; i += blockDim.x) sol[i] = fma(-LU[(size_t)i * m + k], sk, sol[i]);
    __syncthreads();
  }
  if (tid == 0) {
    double dot = 0.0;
    for (int j = 0; j < m; ++j) dot = fma(TNx[j], sol[j], dot);
    out[0] = xNy - dot;
  }
}

int launch_xcy(int64_t n, int64_t m, const double* dN, const double* dT, const double* dS,
               const double* dx, const double* dy, const double* dx0, double* d_work, double* d_out,
               cudaStream_t st) {
  xcy_kernel<<<1, 256, 0, st>>>(n, (int)m, dN, dT, dS, dx, dy, dx0 ? dx0 : dx, d_work, d_out);
  g_launches += 1;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

// ---- TNT = T^T N^-1 T (+ diag(phiinv)) on the device: the matrices enterprise's pta.get_TNT /
// get_phiinv hand to get_mats_fp / get_mats_nmfp (reference fastfp/utils.py:72-76, 97-99), for callers
// that hold only the raw (Nvec, T, phi). Deterministic: the TOA axis is cut into fixed slices, each
// (16 x 16 tile, slice) CTA accumulates its slice in order, a second kernel adds the slices in order.
constexpr int TNT_TILE = 16, TNT_ROWS = 64;

__global__ void __launch_bounds__(256) tnt_partial_kernel(int64_t n, int m, const double* __restrict__ Nvec,
                                                          const double* __restrict__ T, double* __restrict__ part,
                                                          int nsplit) {
  __shared__ double A[TNT_ROWS][TNT_TILE + 1], B[TNT_ROWS][TNT_TILE + 1];
  const int jb = blockIdx.x * TNT_TILE, kb = blockIdx.y * TNT_TILE, sp = blockIdx.z;
  if (kb > jb) return;  // lower triangle of tiles; the reduce kernel mirrors it
  const int tj = threadIdx.x / TNT_TILE, tk = threadIdx.x % TNT_TILE;
  const int64_t per = (n + nsplit - 1) / nsplit, i0 = sp * per, i1 = min(n, i0 + per);
  double acc = 0.0;
  for (int64_t base = i0; base < i1; base += TNT_ROWS) {
    for (int e = threadIdx.x; e < TNT_ROWS * TNT_TILE; e += 256) {
      const int r = e / TNT_TILE, c = e % TNT_TILE;
      const int64_t i = base + r;
      double a = 0.0, b = 0.0;
      if (i < i1) {
        if (jb + c < m) a = T[i * m + jb + c] / Nvec[i];  // (T / Nvec) as enterprise forms it
        if (kb + c < m) b = T[i * m + kb + c];
      }
      A[r][c] = a;
      B[r][c] = b;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < TNT_ROWS; ++r) acc = fma(A[r][tj], B[r][tk], acc);
    __syncthreads();
  }
  if (jb + tj < m && kb + tk < m) part[((size_t)sp * m + jb + tj) * m + kb + tk] = acc;
}

__global__ void tnt_reduce_kernel(int m, const double* __restrict__ part, int nsplit,
                                  const double* __restrict__ phiinv, double* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * m) return;
  const int j = idx / m, k = idx - j * m;
  // tiles (jb, kb <= jb) were computed; take the lower triangle (k <= j) and mirror it, so the result is
  // exactly symmetric (inside a diagonal tile (T_j/N) T_k and (T_k/N) T_j round differently)
  const bool have = k <= j;
  const int jj = have ? j : k, kk = have ? k : j;
  double acc = 0.0;
  for (int sp = 0; sp < nsplit; ++sp) acc += part[((size_t)sp * m + jj) * m + kk];
  if (phiinv && j == k) acc += phiinv[j];
  out[idx] = acc;
}

int launch_tnt(int64_t n, int64_t m, const double* dN, const double* dT, const double* d_phiinv, double* d_part,
               int nsplit, double* d_out, cudaStream_t st) {
  const unsigned nt = (unsigned)((m + TNT_TILE - 1) / TNT_TILE);
  tnt_partial_kernel<<<dim3(nt, nt, (unsigned)nsplit), 256, 0, st>>>(n, (int)m, dN, dT, d_part, nsplit);
  tnt_reduce_kernel<<<(unsigned)((m * m + 255) / 256), 256, 0, st>>>((int)m, d_part, nsplit, d_phiinv, d_out);
  g_launches += 2;
  FFP_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ffp
