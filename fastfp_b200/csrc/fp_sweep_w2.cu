// sweep instantiations: 40 < m <= 80 (one consumer warp covers all rows, 64 frequencies per CTA) -- the m = 72 case.
// 8 consumer + 8 producer warps (512 threads, a 512 x 128 register pool split 168 / 88): each producer warp owns one
// group of 8 frequencies for the whole chunk and evaluates its sincos chains four at a time in lockstep
// (DESIGN.md section 4.2).
#include "fp_sweep_kernel.cuh"
namespace ffp {
#define FFP_SWEEP_CASE_W2(NMBWv) FFP_SWEEP_CASE_W(NMBWv, 2, 1, 32, 8, 8, 168, 88)
int dispatch_sweep_w2(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode, cudaStream_t st) {
  FFP_SWEEP_CASE_W2(6) FFP_SWEEP_CASE_W2(7) FFP_SWEEP_CASE_W2(8) FFP_SWEEP_CASE_W2(9) FFP_SWEEP_CASE_W2(10)
  set_error("no sweep kernel for this configuration (w2)");
  return -3;
}
}  // namespace ffp
