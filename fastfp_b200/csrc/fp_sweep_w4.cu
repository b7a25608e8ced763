// sweep instantiations: 80 < m <= 160 (two warp rows, 32 frequencies per CTA)
#include "fp_sweep_kernel.cuh"
namespace ffp {
int dispatch_sweep_w4(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode, cudaStream_t st) {
  FFP_SWEEP_CASE(6, 2, 2, 16) FFP_SWEEP_CASE(7, 2, 2, 16) FFP_SWEEP_CASE(8, 2, 2, 16) FFP_SWEEP_CASE(9, 2, 2, 16) FFP_SWEEP_CASE(10, 2, 2, 16)
  set_error("no sweep kernel for this configuration (w4)");
  return -3;
}
}  // namespace ffp
