// explicit instantiations of the dense-box sweep with pressure_fix (plain form, no poisson) for NDIM=1 and NDIM=2, all Riemann solvers
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_pfix_plain<1, RIEMANN_LLF>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<1, RIEMANN_EXACT>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<1, RIEMANN_ACOUSTIC>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<1, RIEMANN_HLLC>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<1, RIEMANN_HLL>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<2, RIEMANN_LLF>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<2, RIEMANN_EXACT>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<2, RIEMANN_ACOUSTIC>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<2, RIEMANN_HLLC>(const SweepArgs&, int, cudaStream_t);
template cudaError_t launch_sweep_dense_pfix_plain<2, RIEMANN_HLL>(const SweepArgs&, int, cudaStream_t);
}
