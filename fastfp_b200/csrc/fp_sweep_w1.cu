// sweep instantiations: m <= 40 (one consumer warp covers all rows, 128 frequencies per CTA)
#include "fp_sweep_kernel.cuh"
namespace ffp {
int dispatch_sweep_w1(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode, cudaStream_t st) {
  FFP_SWEEP_CASE(1, 4, 1, 16) FFP_SWEEP_CASE(2, 4, 1, 16) FFP_SWEEP_CASE(3, 4, 1, 16) FFP_SWEEP_CASE(4, 4, 1, 16) FFP_SWEEP_CASE(5, 4, 1, 16)
  set_error("no sweep kernel for this configuration (w1)");
  return -3;
}
}  // namespace ffp
