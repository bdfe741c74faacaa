// explicit instantiations of the dense-box sweep with gravity (poisson) for NDIM=1 and NDIM=2, all Riemann solvers
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_grav<1, RIEMANN_LLF, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<1, RIEMANN_EXACT, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<1, RIEMANN_ACOUSTIC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<1, RIEMANN_HLLC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<1, RIEMANN_HLL, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<2, RIEMANN_LLF, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<2, RIEMANN_EXACT, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<2, RIEMANN_ACOUSTIC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<2, RIEMANN_HLLC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_grav<2, RIEMANN_HLL, false>(const SweepArgs&, int, cudaStream_t);
}
