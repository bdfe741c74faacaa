// explicit instantiation of the 3-D dense-box sweep with pressure_fix (plain form, no poisson), riemann = exact
#include "sweep_dense.cuh"
namespace rgpu {
template cudaError_t launch_sweep_dense_pfix_plain<3, RIEMANN_EXACT>(const SweepArgs&, int, cudaStream_t);
}
