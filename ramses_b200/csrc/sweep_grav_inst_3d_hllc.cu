// explicit instantiations of the 3-D dense-box sweep with gravity (poisson), riemann = hllc: plain and AMR variant
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_grav<3, RIEMANN_HLLC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<3, RIEMANN_HLLC, true>(const SweepArgs&, int, cudaStream_t);
}
