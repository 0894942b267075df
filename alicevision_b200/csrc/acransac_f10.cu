// K10's F10Policy (b200m_acransac_fundamental_distortion_pairs): acransac_kernel<F10Policy> and its launch, in a translation unit
// of their own so that engine.cu's kernels compile as they did without it (see acrk::launch in acransac.cuh).
// block_min, block_sum and bitonic are non-inline __device__ functions of acransac.cuh, defined in engine.cu's translation unit as
// well: here they take names of their own, so that the two objects link (engine.cu's definitions stay as they are).
#define block_min block_min_f10
#define block_sum block_sum_f10
#define bitonic bitonic_f10
#include "acransac.cuh"
#undef block_min
#undef block_sum
#undef bitonic

namespace acrk {

template <>
void launch<F10Policy>(int n_pairs, cudaStream_t st, const Pair* pairs, const double* corr, const float* l10, const uint32_t* mt_state,
                       int mt_stride, long long max_iter, double precision, int skip_on, double* pts_all, uint32_t* idx_all, float* logc_all,
                       unsigned long long* gkeys, uint32_t* gvals, uint32_t* inliers_all, int* trace_all, double* trace_nfa_all, Out* out_all,
                       uint32_t* mt_out) {
  acransac_kernel<F10Policy><<<n_pairs, kThreads, 0, st>>>(pairs, corr, l10, mt_state, mt_stride, max_iter, precision, skip_on, pts_all,
                                                           idx_all, logc_all, gkeys, gvals, inliers_all, trace_all, trace_nfa_all, out_all,
                                                           mt_out);
}

}  // namespace acrk
