// explicit instantiations of the 3-D dense-box sweep with gravity (poisson), riemann = acoustic: plain and AMR variant
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_grav<3, RIEMANN_ACOUSTIC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<3, RIEMANN_ACOUSTIC, true>(const SweepArgs&, int, cudaStream_t);
}
