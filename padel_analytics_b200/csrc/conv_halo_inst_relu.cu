// conv_halo_kernel instantiations of the ReLU epilogue class (see conv_halo_kernel.cuh).
#include "conv_halo_kernel.cuh"

namespace pb {
template HaloKernelFn halo_kernel_lookup<PB_EPI_RELU>(int, int, int);
}  // namespace pb
