/* fastfp_b200 -- C ABI of the B200-native Fp-statistic engine (libfastfp_b200.so).
 *
 * The reference (gabefreedman/fastfp @ 74b0ef8) is pure Python/JAX: it has no FFI of its
 * own. Its hot-path boundary is the Python API
 *     fastfp.utils.get_xCy(Nvec, T, sigma, x, y)                      fastfp/utils.py:27
 *     FastFp.calculate_Fp(fgw, Nvecs, Ts, sigmas)  (+ jax.vmap over fgw) fastfp/fastfp.py:52,
 *                                                                     examples/run_fp.py:63
 *     NMFP.calculate_nmfp(fgw, samples, Nvecs, Ts, TNTs) (+ double vmap) fastfp/nmfp.py:77,
 *                                                                     examples/run_nmfp.py:265-270
 *     RN_container/CURN_container ._powerlaw / .get_phiinv            fastfp/nmfp.py:217-315
 * so the entry points below are exactly what a ctypes binding of those calls needs
 * (INTEGRATION.md shows that binding). Plain pointers and sizes only; no torch / CUDA types.
 *
 * Conventions
 *  - all arithmetic and all arrays are IEEE float64 (reference fastfp/__init__.py:3);
 *  - every function returns 0 on success or a negative FASTFP_ERR_* code; the message is
 *    available from fastfp_last_error() (thread-local); nothing throws across the ABI;
 *  - numerics never raise: NaN/Inf propagate as in the reference (singular M or Sigma,
 *    f <= 0), SURVEY.md section 8(b);
 *  - "host" pointers are ordinary process memory, "dev" pointers are CUDA device memory on
 *    the pack's device; `stream` is a cudaStream_t passed as void* (NULL = default stream).
 *    Calls taking a stream are asynchronous on it unless they copy to host memory, in which
 *    case they synchronise the stream before returning;
 *  - the caller owns every input and output buffer; a pack owns only its own device memory;
 *  - threads: different packs may be used from different host threads concurrently; one pack
 *    carries scratch buffers and a work counter, so calls on the SAME pack must be serialised
 *    by the caller (issuing them on one stream from one thread at a time is enough).
 */
#ifndef FASTFP_B200_H
#define FASTFP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FASTFP_OK 0
#define FASTFP_ERR_INVALID (-1)     /* bad argument (null pointer, negative size, ...) */
#define FASTFP_ERR_CUDA (-2)        /* a CUDA runtime call failed */
#define FASTFP_ERR_UNSUPPORTED (-3) /* shape outside what the kernels were built for */
#define FASTFP_ERR_NOMEM (-4)

/* memory-space flags for fastfp_fp_sweep / fastfp_nmfp_sweep */
#define FASTFP_FREQS_ON_DEVICE 1
#define FASTFP_OUT_ON_DEVICE 2
#define FASTFP_PARAMS_ON_DEVICE 4

typedef struct fastfp_pack fastfp_pack_t; /* opaque: device-resident packed pulsar array */

const char* fastfp_last_error(void);
int fastfp_version(void);
int fastfp_device_count(void);

/* ---- plain Fp ------------------------------------------------------------------------
 * fastfp_pack_create: what FastFp.__init__ (fastfp/fastfp.py:39-45: toas, residuals) plus the
 * (Nvecs, Ts, sigmas) lists of get_mats_fp (fastfp/utils.py:72-78) amount to: the P ragged
 * per-pulsar arrays, copied from host memory and pre-reduced on the device into the packed
 * layout the sweep kernel streams (DESIGN.md section 3).
 *   n[p]            number of TOAs           m[p]   number of basis columns of T_p
 *   toas[p]         (n_p)   seconds          residuals[p] (n_p) seconds
 *   Nvecs[p]        (n_p)   white-noise variances (diagonal N; utils.py:29-31)
 *   Ts[p]           (n_p, m_p) row-major     sigmas[p]    (m_p, m_p) row-major, SPD
 */
int fastfp_pack_create(int device, int P, const int64_t* n, const int64_t* m,
                       const double* const* toas, const double* const* residuals,
                       const double* const* Nvecs, const double* const* Ts,
                       const double* const* sigmas, void* stream, fastfp_pack_t** out);

/* Basis width: m_p <= 2688 columns. One work item of the sweep kernel holds up to 640 G rows; a wider basis is swept
 * as row groups, each one work item, whose b-sums a combine step adds (DESIGN.md section 5h). Above 2688,
 * fastfp_pack_create returns FASTFP_ERR_UNSUPPORTED. Block-diagonal-N packs (m_p <= 632), noise-marginalised packs
 * (m_p <= 640) and residual batches (every m_p <= 640) keep the width of one work item.
 * fastfp_row_groups: the row groups of a basis of width m: their number g (0 if m is outside 1 .. 2688), and with
 * starts non-NULL the first row of each group, starts[0..g] (starts[g] = m). g == 1 for m <= 640. */
int fastfp_row_groups(int64_t m, int64_t* starts);

/* fastfp_fp_sweep: jax.vmap(FastFp.calculate_Fp, in_axes=(0,None,None,None))(freqs, ...)
 * (examples/run_fp.py:63-64; per-frequency body fastfp/fastfp.py:69-92).  out[f] = Fp(freqs[f]),
 * the pulsar sum taken in pulsar order starting from 0 (fastfp.py:71,90). */
int fastfp_fp_sweep(const fastfp_pack_t* pack, const double* freqs, int64_t F, double* out,
                    int flags, void* stream);

/* Which kernel runs the frequency sweep of this pack (the plain-Fp sweep, the Fe sweep, stage A of nmfp). Both
 * compute the same quantities to the same parity bar:
 *   FASTFP_PATH_I8    the tensor-core kernel: Y = G [s c] as an error-free product of 8-bit digit planes
 *                     (wgmma s8 x s8, exact int32 accumulation); takes pulsars with m <= 639 basis columns,
 *                     n <= 16384 TOAs and finite data in packs with a diagonal N (fastfp_pack_set_path(I8) returns
 *                     FASTFP_ERR_UNSUPPORTED unless EVERY pulsar fits);
 *   FASTFP_PATH_MIXED the tensor kernel for the pulsars it takes, the fp64 kernel for the others of the same pack in
 *                     the same sweep (FASTFP_ERR_UNSUPPORTED if it takes none);
 *   FASTFP_PATH_FP64  the fp64 DMMA kernel (always available; block-N packs use it);
 *   FASTFP_PATH_AUTO  (default) the fp64 DMMA kernel, the faster of the two on an H100.
 * fastfp_pack_path returns the path in effect (never AUTO): FP64, I8 (all pulsars) or MIXED (some pulsars on
 * either kernel). */
#define FASTFP_PATH_AUTO 0
#define FASTFP_PATH_FP64 1
#define FASTFP_PATH_I8 2
#define FASTFP_PATH_MIXED 3
int fastfp_pack_set_path(fastfp_pack_t* pack, int path);
int fastfp_pack_path(const fastfp_pack_t* pack);

/* per-pulsar terms 0.5*N^T M^-1 N (fastfp.py:90 before the sum): terms[p*F + f]. Same flags. */
int fastfp_fp_terms(const fastfp_pack_t* pack, const double* freqs, int64_t F, double* terms,
                    int flags, void* stream);

/* ---- Fe-statistic (the reference's to-do, README.md:23) ------------------------------------------------
 * Coherent Earth-term statistic of Ellis, Siemens & Creighton 2012 for S sky positions at once, from the same
 * per-(pulsar, frequency) inner products as Fp (fastfp/fastfp.py:81-88): with antenna patterns F+_p, Fx_p
 *   N = sum_p [F+ N_p ; Fx N_p],  M = sum_p [[F+^2 M_p, F+Fx M_p],[F+Fx M_p, Fx^2 M_p]],  Fe = 1/2 N^T M^-1 N
 * (N_p, M_p as in fastfp.py:83-88; 4x4 general solve with partial pivoting). fplus, fcross: host arrays (S, P)
 * row-major; out: (S, F) row-major. flags as for fastfp_fp_sweep. One sweep + one combine kernel per call.
 * f <= 0 gives NaN at every sky position, as for Fp (the reference's f^(-1/3)). */
int fastfp_fe_sweep(const fastfp_pack_t* pack, const double* freqs, int64_t F, const double* fplus,
                    const double* fcross, int64_t S, double* out, int flags, void* stream);

/* fastfp_fe_skymax: the loudest sky position per frequency of an all-sky scan, without the (S, F) map:
 *   fe_max[f] = max_s Fe(s, f),   sky_index[f] = the s that attains it           (fe_max, sky_index: (F,) each)
 * Every Fe(s, f) is the value fastfp_fe_sweep returns for it, bit for bit. Reduction rule: a NaN loses to every other
 * value; among equal values the lowest sky index wins; a frequency where every position is NaN (e.g. f <= 0) gives
 * fe_max = NaN and sky_index = -1. The result does not depend on how the work is split. fplus, fcross: host arrays
 * (S, P) row-major as for fastfp_fe_sweep; S is limited by device memory only (scratch below).
 * flags as for fastfp_fp_sweep; FASTFP_OUT_ON_DEVICE covers both outputs. Returns FASTFP_ERR_INVALID for a NULL
 * argument, a negative size, an nmfp pack, or S == 0 with F > 0; F == 0 returns FASTFP_OK and writes nothing.
 * Device scratch: the call grows the pack's Fe scratch to 5 P F_batch + 7 S P doubles (one frequency batch of inner
 * products, the antenna patterns and the per-(sky, pulsar) weights; about 750 MB for S = 196 608, P = 68, against
 * 2 S P for the patterns of fastfp_fe_sweep), plus F for host outputs; the pack keeps it, like
 * its other scratch buffers, until fastfp_pack_destroy, so repeated calls allocate nothing. */
int fastfp_fe_skymax(const fastfp_pack_t* pack, const double* freqs, int64_t F, const double* fplus,
                     const double* fcross, int64_t S, double* fe_max, int64_t* sky_index, int flags, void* stream);

/* ---- Fp of a batch of residual realisations ---------------------------------------------------------------
 * False-alarm calibration on simulated noise and injection-recovery studies need Fp over one frequency grid for R
 * residual vectors of the same pulsars, noise model and basis. The residuals enter only through w = C^-1 r, so the R
 * realisations ride along as R extra rows of the G tiles the fp64 kernel already streams, and the sin/cos work is
 * shared (DESIGN.md section 5d).
 * fastfp_pack_set_residuals: residuals[p] is a host array (R, n_p) row-major. The pack keeps the realisations'
 *   packets until the next call or fastfp_pack_destroy; R == 0 releases them. fastfp_pack_bytes counts them. Each
 *   pulsar then needs roundup8(m_p) + roundup8(R) rows of the kernel's 640, so R <= 640 - roundup8(max_p m_p)
 *   (568 at m = 72). Returns FASTFP_ERR_INVALID for a NULL pack or array, R < 0 or an nmfp pack, and
 *   FASTFP_ERR_UNSUPPORTED for a block-N pack (it takes fastfp_pack_set_residuals_blockn) or an R above the limit (the message names the limit and the widest
 *   pulsar). While it runs the call also holds a device staging copy of the realisations, R * sum_p n_p doubles
 *   (3.1 GB at R = 568 for 68 pulsars of 10^4 TOAs), on top of the packets it keeps (sum_p ceil(n_p / CI) * CI *
 *   (4 + MP) doubles, 3.5 GB in that case); the staging copy is freed before it returns.
 * fastfp_fp_sweep_residuals: out is (R, F) row-major, out[k*F + f] = the Fp fastfp_fp_sweep returns for a pack
 *   built with residuals r_k (pulsar sum in pulsar order from 0, same 2x2 rule). The values meet the same parity bar
 *   as fastfp_fp_sweep but are not bit-identical to it: (s|r_k), (c|r_k) come from the MMA instead of the producers'
 *   dot products. It always runs the fp64 DMMA kernel, whatever fastfp_pack_path says. flags as for
 *   fastfp_fp_sweep. FASTFP_ERR_INVALID if no realisations are set; F == 0 writes nothing.
 *   Device scratch: the terms of one frequency batch, R * P * F_batch doubles with F_batch = max(1024,
 *   min(F, 2^27 / (R * P))) (at most 1 GiB unless R * P > 131 072), kept until the realisations are replaced or
 *   released, plus R * F doubles for host outputs in the pack's output buffer, kept until fastfp_pack_destroy. */
int fastfp_pack_set_residuals(fastfp_pack_t* pack, int64_t R, const double* const* residuals, void* stream);
/* fastfp_pack_set_residuals_blockn: the realisations of a block-diagonal N pack (fastfp_pack_create_blockn without
 *   m_fix), for fastfp_fp_sweep_residuals and fastfp_fe_skymax_residuals. Each pulsar's residual packets hold the
 *   basis rows, w_1 .. w_R from row roundup8(m_p) on and the 8 epoch-slot rows last: roundup8(m_p) + roundup8(R) + 8
 *   rows, so R <= 632 - roundup8(max_p m_p) (560 at m = 72). That many rows usually select another kernel family than
 *   the pack's, with another chunk size, so the realisations come in the TOA layout of that chunk size (the layout of
 *   fastfp_pack_create_blockn, built for fastfp_sweep_chunk_toas(roundup8(m_p) + roundup8(R), 1) TOAs per chunk; it
 *   agrees with the pack's layout position by position on every real TOA, and the pack's G rows and 1/N are paired
 *   with it by position):
 *     n[p]            TOA count of that layout, a multiple of its chunk size
 *     residuals[p]    (R, n[p]) row-major, the raw realisations (0 on padding TOAs)
 *     residuals_w[p]  (R, n[p]) row-major, (N^-1 r_k) * Nvec as residuals_w of fastfp_pack_create_blockn
 *     slot_idx[p], slot_val[p]  per TOA of that layout, done_mask[p] per chunk, as for fastfp_pack_create_blockn
 *   R == 0 releases the set. fastfp_pack_bytes counts the packets and the slot masks. Returns FASTFP_ERR_INVALID for a
 *   NULL argument, R < 0, an nmfp pack, a diagonal-N pack (it takes fastfp_pack_set_residuals) or an n[p] that is not a
 *   positive multiple of the chunk size, and FASTFP_ERR_UNSUPPORTED for an R above the limit (the message names the
 *   limit and the widest pulsar). While it runs the call holds device staging copies of both arrays, 2 R * sum_p n_p
 *   doubles, twice the staging of fastfp_pack_set_residuals (5.6 GB at R = 560 for 68 pulsars of 10^4 TOAs), plus the
 *   slot arrays, 12 bytes per TOA; they are freed before it returns. */
int fastfp_pack_set_residuals_blockn(fastfp_pack_t* pack, int64_t R, const int64_t* n, const double* const* residuals,
                                     const double* const* residuals_w, const int32_t* const* slot_idx,
                                     const double* const* slot_val, const unsigned char* const* done_mask,
                                     void* stream);
/* ---- residual batches drawn on the device (DESIGN.md section 5g) -------------------------------------------
 * fastfp_pack_simulate_residuals: sets R realisations r_k = n_k + T Phi^(1/2) zeta_k (+ s_k) of the pack's own noise
 *   model, drawn on the device, as fastfp_pack_set_residuals would set them from the host, for
 *   fastfp_fp_sweep_residuals and fastfp_fe_skymax_residuals. n_k is the white noise sqrt(N_i) z_i, zeta_k the basis
 *   draw, s_k the optional Earth-term signal A_s[k,p] sin(((2 pi) f_k) t) + A_c[k,p] cos(((2 pi) f_k) t), the template
 *   of the sweep, phase rounding and sincos rule included. The realisations are never formed: with w = C^-1 r and
 *   C^-1 T Phi = N^-1 T Sigma^-1 the sweep needs w_k = N^-1 n_k - G^T (G n_k - L^-1 (sqrt(phiinv) o zeta_k)) with the
 *   pack's G and Sigma = L L^T, so the draw has covariance exactly N + T Phi T^T = C, timing-model columns included
 *   (phiinv = 1e-40 gives them a negligible weight; phiinv = 0, a flat prior, contributes nothing).
 *     seed     >= 0; first >= 0: the global index of the first realisation (row k is realisation first + k)
 *     phiinv[p] host array (m_p): the 1/phi that went into sigma_p; finite and >= 0
 *     sig_freq host array (R) and sig_amp host array (R, P, 2) of (A_s, A_c), or both NULL: no signal
 *     flags    0, or FASTFP_SIM_NO_NOISE: the signal alone
 *   Random stream: Philox4x64-10 with key (seed, 0) and counter (q, k, p, tag), k = first + row the global realisation
 *   index, p the pulsar, tag 0 for the white noise (normal number = the pulsar's original TOA index), 1 for the ECORR
 *   epoch draws of fastfp_pack_simulate_residuals_blockn (normal number = epoch, in the caller's slice order) and 2
 *   for the basis columns (normal number = column j). Counter block q gives normals 4q .. 4q+3: each of its four
 *   64-bit words x becomes the uniform ((x >> 11) + 0.5) 2^-53 in (0, 1] (never 0; the largest word rounds to
 *   1), and Box-Muller maps (u0, u1) to
 *   sqrt(-2 ln u0) (cos, sin)(2 pi u1) and (u2, u3) likewise. So realisation k is the same whatever R, first or pass
 *   split produced it; np.random.Philox(key=[seed, 0], counter=[q - 1, k, p, tag]).random_raw(4) gives block q, q >= 1
 *   (fastfp_b200/sim.py is the host reference).
 *   Limits, the R == 0 release, the refusal of an nmfp pack (FASTFP_ERR_INVALID) and of a block-N pack
 *   (FASTFP_ERR_UNSUPPORTED) as for fastfp_pack_set_residuals; FASTFP_ERR_INVALID also for a negative seed or first,
 *   a signal given by half, an unknown flag or a phiinv entry that is negative or not finite. Device staging as for
 *   fastfp_pack_set_residuals: R * sum_p n_p doubles, freed before it returns; the R x m draws of the basis need no
 *   more, and nothing crosses PCIe per realisation but the signal (3 P + 1 doubles). */
#define FASTFP_SIM_NO_NOISE 1
int fastfp_pack_simulate_residuals(fastfp_pack_t* pack, int64_t R, int64_t seed, int64_t first,
                                   const double* const* phiinv, const double* sig_freq, const double* sig_amp,
                                   int flags, void* stream);
/* fastfp_pack_simulate_residuals_blockn: the same for a block-diagonal N pack, whose n_k also holds the ECORR draws
 *   sqrt(j_e) eta_e on every TOA of epoch e, and whose N^-1 n_k is applied on the device (Sherman-Morrison). n,
 *   slot_idx, slot_val and done_mask are the residual layout of fastfp_pack_set_residuals_blockn; per pulsar also
 *     toa_index[p]  per position of that layout, the original TOA index (-1 on padding)
 *     epoch[p]      per position, the epoch (index into the caller's slices; -1 outside any epoch and on padding);
 *                   every epoch one contiguous run of positions
 *     sqrt_j[p], beta[p]  per epoch: sqrt(j_e) and beta_e = j_e / (1 + j_e sum_e 1/Nvec)
 *   Refusals as for fastfp_pack_set_residuals_blockn plus those of fastfp_pack_simulate_residuals, and
 *   FASTFP_ERR_INVALID for an epoch or TOA index out of range, an epoch split in two runs, or a sqrt_j / beta that is
 *   not finite (sqrt_j < 0). Device staging: 2 R * sum_p n_p doubles (n_k and (N^-1 n_k) * Nvec), freed before it
 *   returns, as for fastfp_pack_set_residuals_blockn. */
int fastfp_pack_simulate_residuals_blockn(fastfp_pack_t* pack, int64_t R, int64_t seed, int64_t first,
                                          const double* const* phiinv, const double* sig_freq, const double* sig_amp,
                                          const int64_t* n, const int32_t* const* slot_idx,
                                          const double* const* slot_val, const unsigned char* const* done_mask,
                                          const int32_t* const* toa_index, const int32_t* const* epoch,
                                          const double* const* sqrt_j, const double* const* beta, int flags,
                                          void* stream);
int fastfp_fp_sweep_residuals(const fastfp_pack_t* pack, const double* freqs, int64_t F, double* out, int flags,
                              void* stream);

/* fastfp_fe_skymax_residuals: the sky-maximised Fe of fastfp_fe_skymax for each realisation set by
 *   fastfp_pack_set_residuals: fe_max[k*F + f] = max_s Fe_k(s, f), sky_index[k*F + f] = the s that attains it
 *   (fe_max, sky_index: (R, F) row-major), with the reduction rule of fastfp_fe_skymax (NaN loses, ties go to the
 *   lowest index, an all-NaN column gives NaN and -1). The false-alarm threshold of an all-sky search has no closed
 *   form; this is the scan of simulated realisations that calibrates it. The values meet the parity bar of
 *   fastfp_fe_skymax but are not bit-identical to it: (s|r_k), (c|r_k) come from the sweep's MMA, N_k from an MMA over
 *   the pulsars, and the 4x4 solve multiplies by reciprocal pivots (DESIGN.md section 5e). It always runs the fp64
 *   kernel, whatever fastfp_pack_path says. fplus, fcross: host arrays (S, P) row-major. flags as for fastfp_fp_sweep;
 *   FASTFP_OUT_ON_DEVICE covers both outputs. Returns FASTFP_ERR_INVALID for a NULL argument, a negative size, an nmfp
 *   pack, a pack with no realisations set, or S == 0 with F > 0; F == 0 returns
 *   FASTFP_OK and writes nothing.
 *   Device scratch, grown on demand and kept until fastfp_pack_destroy: the realisations' inner products of one
 *   frequency batch, 2 R P F_batch doubles in the residual terms buffer (kept until the realisations are replaced or
 *   released), and in the pack's Fe scratch 3 P F_batch + 2 S P doubles, plus R F for host outputs and, when the sky is
 *   split across CTAs (a single batch of few frequencies), 2 R F per sky chunk; F_batch = max(1024, min(F, 2^27 /
 *   ((2R + 3) P))). About 1.1 GB at R = 248, P = 45, F = 10^4, S = 3072. R F doubles for host outputs live in the
 *   pack's output buffer as for fastfp_fp_sweep_residuals. */
int fastfp_fe_skymax_residuals(const fastfp_pack_t* pack, const double* freqs, int64_t F, const double* fplus,
                               const double* fcross, int64_t S, double* fe_max, int64_t* sky_index, int flags,
                               void* stream);

/* ---- noise-marginalised Fp -----------------------------------------------------------
 * fastfp_nmfp_pack_create: NMFP.__init__ (fastfp/nmfp.py:45-51) plus the (TNTs, Nvecs, Ts)
 * of get_mats_nmfp (fastfp/utils.py:97-101). Sigma_d = TNT + diag(phiinv_d) is formed per
 * draw (nmfp.py:58-74). The phi layouts of nmfp.py:264-292 are [tm | (ecorr) | rn(+curn)]:
 * the first m_fix[p] entries do not depend on the draw (phiinv_fix[p], length m_fix[p]);
 * the remaining m_var[p] = m[p] - m_fix[p] entries come per draw.
 */
int fastfp_nmfp_pack_create(int device, int P, const int64_t* n, const int64_t* m,
                            const double* const* toas, const double* const* residuals,
                            const double* const* Nvecs, const double* const* Ts,
                            const double* const* TNTs, const int64_t* m_fix,
                            const double* const* phiinv_fix, void* stream,
                            fastfp_pack_t** out);

/* fastfp_nmfp_sweep: vmap_g(vmap_f(nmfp))(freqs, samples, ...) of examples/run_nmfp.py:265-270.
 * phiinv_var: (D, sum_p m_var[p]) row-major, draw d / pulsar p / varying column k at
 * d*ld + off_p + k with off_p = sum_{q<p} m_var[q] and ld = sum_p m_var[p].
 * out: (D, F) row-major, draw-major like the reference. */
int fastfp_nmfp_sweep(const fastfp_pack_t* pack, const double* freqs, int64_t F,
                      const double* phiinv_var, int64_t D, double* out, int flags, void* stream);

/* The two halves of fastfp_nmfp_sweep as separate calls, for callers that shard the work in two dimensions over
 * several GPUs (fastfp_b200/parallel.py::sharded_nmfp): stage A -- everything that depends on the frequency but not on
 * the draw (nmfp.py:103-113: the sin/cos templates through T^T N^-1 and the draw-independent block of Sigma) -- is
 * computed for a SLICE of the frequency grid per GPU and all-gathered; factor + stage B (nmfp.py:58-74, 114-119) then
 * run per GPU for its draws on all frequencies. All pointers are device memory on the pack's device.
 *   fastfp_nmfp_tile_sizes  doubles per 32-frequency tile (all pulsars) of the two stage-A outputs
 *   fastfp_nmfp_stage_a     z (ceil(F/32) * z_per_tile) and a (ceil(F/32) * a_per_tile) for F frequencies
 *   fastfp_nmfp_stage_b     z / a hold consecutive blocks of tiles_per_block tiles each (one block per gathered
 *                           slice; even unless there is one block), together the ceil(F/32) tiles of freqs;
 *                           out: (D, F) row-major */
int fastfp_nmfp_tile_sizes(const fastfp_pack_t* pack, int64_t* z_per_tile, int64_t* a_per_tile);
int fastfp_nmfp_stage_a(const fastfp_pack_t* pack, const double* freqs_dev, int64_t F, double* z_dev, double* a_dev,
                        void* stream);
int fastfp_nmfp_stage_b(const fastfp_pack_t* pack, const double* freqs_dev, int64_t F, const double* z_dev,
                        const double* a_dev, int64_t tiles_per_block, const double* phiinv_var_dev, int64_t D,
                        double* out_dev, void* stream);

/* fastfp_powerlaw_phiinv: RN_container.get_phiinv for the varying block (nmfp.py:226-234,
 * 247/275 CURN add, 305-315 reciprocal), for D draws and P pulsars at once, on the device.
 *   Ffreqs[p]      (m_var[p]) repeat(k/Tspan,2) of pulsar p (host)
 *   log10_A, gamma (D, P) row-major red-noise parameters
 *   curn_Ffreqs    (ncurn) or NULL; curn_log10_A, curn_gamma (D) -- added onto the leading
 *                  ncurn entries of every pulsar (nmfp.py:275)
 *   phiinv_var     output, device memory, layout as fastfp_nmfp_sweep expects. */
int fastfp_powerlaw_phiinv(const fastfp_pack_t* pack, const double* const* Ffreqs,
                           const double* log10_A, const double* gamma, int64_t D,
                           const double* curn_Ffreqs, int64_t ncurn, const double* curn_log10_A,
                           const double* curn_gamma, double* phiinv_var_dev, void* stream);

/* ---- block-diagonal N (EcorrKernelNoise) ------------------------------------------------------
 * The reference leaves this case open ("does not apply ... where N is block-diagonal",
 * fastfp/utils.py:29-31; README to-do). N = diag(Nvec) + sum_e j_e 1_e 1_e^T over epochs of TOAs.
 * The host side (fastfp_b200/blockn.py) lays the TOAs out in chunks of fastfp_sweep_chunk_toas(m, 1)
 * so that every group of 4 TOAs belongs to one epoch, applies the Sherman-Morrison N^-1 to T and r,
 * and passes per TOA the epoch slot (0..7 inside its chunk, -1 = none) with sqrt(beta_e)/Nvec_i,
 * beta_e = j_e / (1 + j_e sum_e 1/Nvec), and per chunk the mask of slots whose epoch ends there.
 *   residuals_w[p] = (N^-1 r) * Nvec,  Ts[p] = (N^-1 T) * Nvec row-wise,  Nvecs[p] = diagonal part
 *   (inf on padding TOAs);  mats[p] = sigma_p (m_fix == NULL: plain Fp) or TNT_p (nmfp, with m_fix /
 *   phiinv_fix as in fastfp_nmfp_pack_create), both formed with the block N.
 * The resulting pack is used with fastfp_fp_sweep / fastfp_nmfp_sweep unchanged; a plain-Fp one takes residual
 * batches through fastfp_pack_set_residuals_blockn.
 * The epoch slots take 8 rows of the G tile after the basis rows (roundup8(m) + 8 in all), so a block-N pulsar
 * has m <= 632: fastfp_sweep_chunk_toas(m, 1) returns 0 above that and fastfp_pack_create_blockn returns
 * FASTFP_ERR_UNSUPPORTED. */
int fastfp_sweep_chunk_toas(int64_t m, int blockn);
int fastfp_pack_create_blockn(int device, int P, const int64_t* n, const int64_t* m,
                              const double* const* toas, const double* const* residuals,
                              const double* const* residuals_w, const double* const* Nvecs,
                              const double* const* Ts, const double* const* mats,
                              const int32_t* const* slot_idx, const double* const* slot_val,
                              const unsigned char* const* done_mask, const int64_t* m_fix,
                              const double* const* phiinv_fix, void* stream, fastfp_pack_t** out);

void fastfp_pack_destroy(fastfp_pack_t* pack);
int64_t fastfp_pack_bytes(const fastfp_pack_t* pack);    /* device bytes held */
int fastfp_pack_num_pulsars(const fastfp_pack_t* pack);
int64_t fastfp_pack_mvar_total(const fastfp_pack_t* pack); /* sum_p m_var[p] (nmfp packs) */
/* Status of the one-time Cholesky of Sigma_p (plain Fp) or of its draw-independent block (nmfp):
 * info[p] = 0, or j+1 when pivot j was not positive -- Sigma_p is then not numerically symmetric positive
 * definite (the sweep path factorises Sigma = L L^T and reads its lower triangle; the reference's
 * jnp.linalg.solve, fastfp/utils.py:54, accepts any non-singular matrix, and so does fastfp_xcy). The
 * statistic of such a pulsar is NaN, as a singular Sigma gives in the reference; nothing is raised.
 * Returns the number of pulsars with info != 0 (>= 0), or a negative error code; info may be NULL. */
int fastfp_pack_factor_info(const fastfp_pack_t* pack, int32_t* info);
/* 64-bit content hash of a host buffer (multi-threaded for large buffers; deterministic): what the Python
 * mirror uses to key its pack cache on every byte of the caller's arrays. */
uint64_t fastfp_hash64(const void* data, int64_t nbytes, uint64_t seed);
/* the same for n buffers in one call (out[i] == fastfp_hash64(ptrs[i], nbytes[i], seeds[i])): the pieces of all
 * buffers share one set of threads, so a list of many medium-sized arrays hashes at memory bandwidth. */
int fastfp_hash64_many(const void* const* ptrs, const int64_t* nbytes, int32_t n, const uint64_t* seeds, uint64_t* out);
int64_t fastfp_kernel_launches(void); /* kernels launched by this library so far (process-wide) */
int64_t fastfp_device_bytes(void);    /* device memory this library holds now, in bytes (process-wide) */
/* measurement aid: with enable != 0 every later fastfp_nmfp_sweep on this pack brackets its three
 * stages with CUDA events on the caller's stream and synchronises at the end; fastfp_nmfp_stage_ms
 * then returns the milliseconds of the last sweep {stage A sweep kernel + clears, per-draw factor
 * kernel, stage B kernel}. Off by default (no synchronisation on the normal path). */
int fastfp_nmfp_stage_timing(fastfp_pack_t* pack, int enable);
int fastfp_nmfp_stage_ms(const fastfp_pack_t* pack, double* ms3);

/* ---- single inner product --------------------------------------------------------------
 * fastfp_xcy: fastfp.utils.get_xCy (fastfp/utils.py:49-54) on the device: host arrays in,
 * x^T C^-1 y out, general (LU, partial pivoting) Sigma solve like jnp.linalg.solve. */
int fastfp_xcy(int device, int64_t n, int64_t m, const double* Nvec, const double* T,
               const double* sigma, const double* x, const double* y, double* out, void* stream);
/* fastfp_tnt: TNT = T^T N^-1 T for diagonal N (host arrays; out is (m, m) row-major), plus
 * diag(phiinv) when phiinv is not NULL -- i.e. the Sigma of get_mats_fp (fastfp/utils.py:76) or the
 * TNT of get_mats_nmfp (fastfp/utils.py:97) for callers that hold only the raw basis. Deterministic. */
int fastfp_tnt(int device, int64_t n, int64_t m, const double* Nvec, const double* T,
               const double* phiinv, double* out, void* stream);
/* the same inner product for a block-diagonal N = diag(Nvec) + epoch blocks: xw = (N^-1 x) * Nvec and
 * yw = (N^-1 y) * Nvec are prepared on the host (Sherman-Morrison), x is the raw vector; sigma is the
 * block-N Sigma. (The reference's get_xCy excludes this case, fastfp/utils.py:29-31.) */
int fastfp_xcy_blockn(int device, int64_t n, int64_t m, const double* Nvec, const double* T,
                      const double* sigma, const double* x, const double* xw, const double* yw,
                      double* out, void* stream);

/* ---- measurement helper ----------------------------------------------------------------
 * fastfp_fp64_peak: times a dependent-chain-free DFMA loop (kind 0) or DMMA m8n8k4 loop
 * (kind 1), or both interleaved (kind 2), on the device and returns TFLOP/s; bench.py uses
 * kind 1 as the measured fp64-pipe denominator (MEASURED_PEAKS.json has no fp64 figure). Kinds 3-12
 * are the kernel-design probes of csrc/microbench.cu; 13-15 run the sweep kernel's warp
 * specialisation (8 DMMA warps + 16 DFMA warps) on registers only; 16 = legacy INT8 mma.sync rate
 * (reported as 2 x MAC/s in the same unit); 17 = s8 wgmma m64n256k32 on two warpgroups (the INT8 tensor peak, TOP/s);
 * 18 = the tensor sweep's own stage (28 plane products, two warpgroups of m64n32k32); 19-24 the fp64 MMA shapes and
 * consumer tiles; 22 / 25 the warp specialisation on m16n8k4 at the 8 + 16 and 8 + 8 warp splits. */
int fastfp_fp64_peak(int device, int kind, int iters, double* tflops, double* ms);

#ifdef __cplusplus
}
#endif
#endif /* FASTFP_B200_H */
