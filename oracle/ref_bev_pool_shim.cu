// oracle/ref_bev_pool_shim.cu — TEST INFRASTRUCTURE ONLY (GPU-side oracle for BEVPoolV2).
//
// Exports the reference's own BEVPoolV2 launchers with C linkage, for the golden fixture and the timing script:
//   TensorRT/plugin/bev_pool_v2/bevPoolKernel.h               (declared there; the TensorRT plugin's forward kernels)
//   third_party/bev_mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu  (the training backward; its launcher is declared by
//                                                                  bev_pool.cpp, restated below)
// Both translation units are compiled unmodified from where they lie in the reference tree (oracle/bev_pool.mk). This
// file contains no arithmetic. The mmdet3d launchers run on the legacy default stream, so their exports synchronise.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "bevPoolKernel.h"

void bev_pool_v2_grad(int c, int n_intervals, const float *out_grad, const float *depth, const float *feat,
                      const int *ranks_depth, const int *ranks_feat, const int *ranks_bev, const int *interval_starts,
                      const int *interval_lengths, float *depth_grad, float *feat_grad);

extern "C" {

// dtype: 0 f32, 1 f16 (bev_pool_v2_kernel<__half>, BEVPoolV2TRT), 2 f16 as half2 (BEVPoolV2TRT2; c must be even).
// out_numel = elements of the output, which the launcher zeroes first.
void ref_bev_pool(int dtype, int c, int n_intervals, int out_numel, const void *depth, const void *feat,
                  const int *ranks_depth, const int *ranks_feat, const int *ranks_bev, const int *interval_starts,
                  const int *interval_lengths, void *out, void *stream) {
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == 0)
    bev_pool_v2<float>(c, n_intervals, out_numel, (const float *)depth, (const float *)feat, ranks_depth, ranks_feat,
                       ranks_bev, interval_starts, interval_lengths, (float *)out, s);
  else if (dtype == 1)
    bev_pool_v2<__half>(c, n_intervals, out_numel, (const __half *)depth, (const __half *)feat, ranks_depth,
                        ranks_feat, ranks_bev, interval_starts, interval_lengths, (__half *)out, s);
  else
    bev_pool_v2_h2(c, n_intervals, out_numel, (const __half *)depth, (const __half2 *)feat, ranks_depth, ranks_feat,
                   ranks_bev, interval_starts, interval_lengths, (__half2 *)out, s);
}

void ref_bev_pool_int8(int c, int n_intervals, int out_numel, const void *depth, float scale_d, const void *feat,
                       float scale_f, const int *ranks_depth, const int *ranks_feat, const int *ranks_bev,
                       const int *interval_starts, const int *interval_lengths, void *out, float scale_o, void *stream) {
  bev_pool_v2_int8(c, n_intervals, out_numel, (const int8_t *)depth, scale_d, (const int8_4 *)feat, scale_f,
                   ranks_depth, ranks_feat, ranks_bev, interval_starts, interval_lengths, (int8_4 *)out, scale_o,
                   (cudaStream_t)stream);
}

// mmdet3d's training backward (QuickCumsumCuda): depth_grad / feat_grad must be zeroed by the caller, and the
// intervals are those of the points regrouped by ranks_feat, as QuickCumsumCuda.backward builds them.
void ref_bev_pool_backward_f32(int c, int n_intervals, const float *out_grad, const float *depth, const float *feat,
                               const int *ranks_depth, const int *ranks_feat, const int *ranks_bev,
                               const int *interval_starts, const int *interval_lengths, float *depth_grad,
                               float *feat_grad) {
  bev_pool_v2_grad(c, n_intervals, out_grad, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts,
                   interval_lengths, depth_grad, feat_grad);
  cudaDeviceSynchronize();
}

}  // extern "C"
