// sweep instantiations: 160 < m <= 320 (four warp rows, 16 frequencies per CTA)
#include "fp_sweep_kernel.cuh"
namespace ffp {
int dispatch_sweep_wide(const fastfp_pack* pk, const GroupView& g, const SweepArgs& a, SweepMode mode,
                        cudaStream_t st) {
  FFP_SWEEP_CASE(6, 2, 4, 16) FFP_SWEEP_CASE(7, 2, 4, 16) FFP_SWEEP_CASE(8, 2, 4, 16) FFP_SWEEP_CASE(9, 2, 4, 16) FFP_SWEEP_CASE(10, 2, 4, 16)
  set_error("no sweep kernel for this configuration (wide)");
  return -3;
}
}  // namespace ffp
