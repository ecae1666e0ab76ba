// conv_halo_kernel instantiations of the run-time epilogue class (see conv_halo_kernel.cuh).
#include "conv_halo_kernel.cuh"

namespace pb {
template HaloKernelFn halo_kernel_lookup<PB_EPI_GENERIC>(int, int, int);
}  // namespace pb
