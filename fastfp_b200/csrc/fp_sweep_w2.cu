// sweep instantiations: 40 < m <= 80 (one consumer warp covers all rows, 64 frequencies per CTA) -- the m = 72 case
#include "fp_sweep_kernel.cuh"
namespace ffp {
int dispatch_sweep_w2(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode, cudaStream_t st) {
  FFP_SWEEP_CASE(6, 2, 1, 32) FFP_SWEEP_CASE(7, 2, 1, 32) FFP_SWEEP_CASE(8, 2, 1, 32) FFP_SWEEP_CASE(9, 2, 1, 32) FFP_SWEEP_CASE(10, 2, 1, 32)
  set_error("no sweep kernel for this configuration (w2)");
  return -3;
}
}  // namespace ffp
