// sweep instantiations: 320 < m <= 640 (eight warp rows, 8 frequencies per CTA, chunks of 8 TOAs)
#include "fp_sweep_kernel.cuh"
namespace ffp {
int dispatch_sweep_xwide(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode,
                         cudaStream_t st) {
  FFP_SWEEP_CASE(6, 2, 8, 8) FFP_SWEEP_CASE(7, 2, 8, 8) FFP_SWEEP_CASE(8, 2, 8, 8) FFP_SWEEP_CASE(9, 2, 8, 8) FFP_SWEEP_CASE(10, 2, 8, 8)
  set_error("no sweep kernel for this configuration (xwide)");
  return -3;
}
}  // namespace ffp
