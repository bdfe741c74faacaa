// explicit instantiations of the 3-D dense-box sweep with pressure_fix (AMR variant), riemann = hllc: without and with poisson
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_pfix<RIEMANN_HLLC, false>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix<RIEMANN_HLLC, true>(const SweepArgs&, int, cudaStream_t);
}
