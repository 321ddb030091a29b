/*
 * b200_bev_ops.h — C ABI of libb200_bev_ops.so: BEVFormer's attention-sampling hot path for NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for the three TensorRT plugins of DerryHub/BEVFormer_tensorrt that sit on that path.
 * Every entry point replaces one launcher of the reference (the level directly under IPluginV2DynamicExt::enqueue)
 * and keeps its argument order and meaning; `file:line` below are relative to the reference repository.
 *
 * Conventions (all entry points)
 *   - All data pointers are DEVICE pointers owned by the caller (TensorRT / PyTorch); nothing is allocated, freed
 *     or retained. `stream` is a cudaStream_t passed as void*; launches are asynchronous on it, no syncs.
 *   - Return value: B200_OK (0) on success; non-zero status otherwise. Never aborts/exits the process (the reference
 *     ASSERT()s -> abort(), TensorRT/common/helper.h:43-49, and printf()s launch errors, …Kernel.cu:1124-1127).
 *     B200_ERR_UNSUPPORTED == 1 matches enqueue()'s "return 1" for an unsupported dtype (…Plugin.cpp:136-139).
 *   - No CPU fallback exists: without a CUDA device the launch fails and the status says so.
 */
#ifndef B200_BEV_OPS_H
#define B200_BEV_OPS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  B200_OK = 0,
  B200_ERR_UNSUPPORTED = 1, /* dtype / format / shape combination not implemented */
  B200_ERR_BAD_PARAM = 2,   /* null pointer, non-positive dimension, size overflow, misalignment */
  B200_ERR_LAUNCH = 3       /* CUDA reported an error at launch (cudaGetLastError) */
};

/* Library / build identification: "b200_bev_ops <version> sm_90a". */
const char *b200_bev_ops_version(void);
/* Text for a status code. */
const char *b200_status_string(int status);
/* Number of kernels this library has launched since load (bench.py's gpu_launches claim is counted here). */
unsigned long long b200_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------
 * Multi-scale deformable attention (plugin MultiScaleDeformableAttnTRT / …TRT2)
 *
 *   value            [batch, spatial_size, num_heads, channels]      levels concatenated along spatial_size
 *   spatial_shapes   int32 [num_levels, 2] (h, w), device memory
 *   reference_points [batch, num_query, 1, 2*points_per_group]       normalised (x, y) per group (Z anchor)
 *   sampling_offsets [batch, num_query, num_heads, num_levels*num_point*2]   pixels of that level, (x, y) innermost
 *   attn_weight      [batch, num_query, num_heads, num_levels*num_point]     PRE-softmax logits
 *   out              [batch, num_query, num_heads, channels]
 *
 * Semantics = the reference FP32 kernel (…/multiScaleDeformableAttnKernel.cu:611-688, :133-178): softmax over
 * all num_levels*num_point logits, loc = fma(ref, size, off) - 0.5 (bit-exact index arithmetic), zero-padded bilinear
 * taps. The FP16 entry stores FP16 but evaluates indices and accumulates in FP32 (the reference's __half kernels do
 * the coordinate math in half precision, :740-756; that loss is deliberately not reproduced).
 * ---------------------------------------------------------------------------------------------------------- */

/* replaces ms_deformable_im2col_cuda<float>   — …/multiScaleDeformableAttnKernel.h:12-19, .cu:1106-1128 */
int b200_msda_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                  const float *sampling_offsets, const float *attn_weight, int batch, int spatial_size, int num_heads,
                  int channels, int num_levels, int num_query, int num_point, int points_per_group, float *out,
                  void *stream);

/* replaces ms_deformable_im2col_cuda<__half>  — …Kernel.h:12-19 (T=__half), .cu:1130-1149; pointers are __half* */
int b200_msda_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                  const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size, int num_heads,
                  int channels, int num_levels, int num_query, int num_point, int points_per_group, void *out,
                  void *stream);

/* replaces ms_deformable_im2col_cuda_h2        — …Kernel.h:21-27, .cu:1151-1169. Same memory layout as _f16
 * (__half2 is a reinterpretation); needs even `channels` like the reference (…Plugin.cpp:240-245). */
int b200_msda_f16_h2(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                     const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                     int num_heads, int channels, int num_levels, int num_query, int num_point, int points_per_group,
                     void *out, void *stream);

/* BF16 (beyond the reference, which has no BF16 plugin): value, sampling_offsets, attn_weight and out are
 * __nv_bfloat16; reference_points are FP32 (bf16's 8 significant bits would move a normalised point by up to 2^-9 of
 * the level's extent). Arithmetic = the FP16 entry's exact mode: every bf16 element widened to FP32 exactly, FP32 index
 * arithmetic and accumulation, one rounding of the result (round to nearest even). Same kernel selection and launch
 * shapes as b200_msda_f16; b200_msda_set_f16_mode / _set_f16_path do not apply. */
int b200_msda_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                   const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size, int num_heads,
                   int channels, int num_levels, int num_query, int num_point, int points_per_group, void *out,
                   void *stream);

/* replaces ms_deformable_im2col_cuda_int8<float> / <__half2> — …Kernel.h:29-38, .cu:1172-1218.
 * value / offsets / attn_weight / out are int8 with per-tensor scales (real = q * scale, TensorRT PTQ convention,
 * …Plugin.cpp:75-77); reference_points are float (ref_is_half == 0) or __half (ref_is_half != 0).
 * Needs channels % 4 == 0 and num_point % 4 == 0 like the reference (…Plugin.cpp:151-156).
 * Arithmetic: in-register dequantisation, FP32 evaluation, one requantisation of the result with
 * round-half-away-from-zero and saturation (T2int8, .cu:51-55). */
int b200_msda_i8(const int8_t *value, float scale_value, const int32_t *spatial_shapes, const void *reference_points,
                 int ref_is_half, const int8_t *sampling_offsets, float scale_offset, const int8_t *attn_weight,
                 float scale_weight, int batch, int spatial_size, int num_heads, int channels, int num_levels,
                 int num_query, int num_point, int points_per_group, int8_t *out, float scale_out, void *stream);

/* Fused spatial-cross-attention sampling (beyond the reference's plugin set; SURVEY.md §8(f)-1): MSDA followed by the
 * bev_mask-weighted sum over cameras that SpatialCrossAttention applies to the plugin output
 * (det2trt/models/modules/spatial_cross_attention.py:270 — slots = (queries * bev_mask).sum(0)):
 *     accum[q, m*channels + c] += bev_mask[b, q] * MSDA(value, …)[b, q, m, c]        (fp32 accumulator, += semantics)
 * The per-camera output [batch, num_query, heads, channels] is never written; cameras that do not see a query add
 * nothing. bev_mask: float [batch, num_query]; accum: float [num_query, num_heads*channels], zeroed by the caller.
 * Needs channels == 32, num_point % 4 == 0, points_per_group in {1,2,4} (returns B200_ERR_UNSUPPORTED otherwise). */
int b200_msda_sca_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                      const float *sampling_offsets, const float *attn_weight, const float *bev_mask, int batch,
                      int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                      int points_per_group, float *accum, void *stream);
int b200_msda_sca_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                      const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                      int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                      int points_per_group, float *accum, void *stream);
/* BF16 value / offsets / logits, FP32 reference points (see b200_msda_bf16). */
int b200_msda_sca_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                       const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                       int spatial_size, int num_heads, int channels, int num_levels, int num_query, int num_point,
                       int points_per_group, float *accum, void *stream);

/* Camera-shared form of the same fused op. SpatialCrossAttention repeats the BEV query for every camera before the
 * sampling_offsets / attention_weights Linear layers (spatial_cross_attention.py:254 `query.repeat(num_cams, 1, 1)`), so
 * the [batch, ...] offsets and logits the plugin receives are `batch` identical copies. Here they are passed once:
 *     sampling_offsets [num_query, heads, levels*points*2],  attn_weight [num_query, heads, levels*points]
 *     value [batch, keys, heads, channels], reference_points [batch, num_query, 1, 2*G], bev_mask [batch, num_query]
 *     slots[q, m*channels + c] = sum_b bev_mask[b, q] * MSDA(value[b], ref[b], offsets, logits)[q, m, c]   (plain store)
 * One item per (query, head): the softmax is evaluated once, the cameras that see the query are looped in registers and
 * every slot is written exactly once (no atomics, no pre-zeroed accumulator; queries no camera sees get zeros). The
 * two Linear layers upstream shrink by `batch`x and 5/6 of the offsets/logits bytes disappear. Same shape limits. */
int b200_msda_sca_shared_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                             const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                             int batch, int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                             int num_point, int points_per_group, float *slots, void *stream);
int b200_msda_sca_shared_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                             const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                             int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                             int num_point, int points_per_group, float *slots, void *stream);
int b200_msda_sca_shared_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                              const void *sampling_offsets, const void *attn_weight, const float *bev_mask, int batch,
                              int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                              int num_point, int points_per_group, float *slots, void *stream);

/* ---- Second-generation INT8 MSDA path (csrc/msda_v2.cu): channels == 32, 16 <= num_levels*num_point <= 32 ----
 * Same operator, same semantics and argument meaning as b200_msda_i8, with one addition to the signature: the caller
 * lends a WORKSPACE (TensorRT: IPluginV2DynamicExt::getWorkspaceSize / enqueue's `workspace`; the reference's plugin
 * asks for 0 bytes, …Plugin.cpp:64-69). Its size depends on tensor DIMENSIONS only (a bound: 3 * spatial_size 64-byte
 * entries per camera and head — at base shapes 97 MB of it are touched); spatial_shapes stays the device tensor the
 * reference plugin receives, the packed-stack plan is evaluated on the device.
 * Two launches per call: (1) a pack pre-pass re-lays `value` into per-(camera, head) column-pair entries with the two
 * image rows interleaved per channel (value tiles staged through shared memory by TMA bulk copies); (2) the gather:
 * persistent CTAs bound to one (camera, head) slab of the packed stack, the coarsest levels of the slab resident in
 * shared memory (TMA bulk copies; b200_msda_set_i8_resident_bytes, default 128 KiB); a bilinear sample is one 128-byte
 * run, one 16-byte load per lane (shared memory for resident levels, L1/L2 otherwise), accumulated with dp2a against
 * 16-bit fixed-point tap weights in int32, one requantisation (T2int8). Index arithmetic is the round-1 kernel's
 * (FP32, bit-exact).
 * `trace_records` (optional, may be NULL): the gather kernel's own sampling-index records, as in b200_msda_i8_trace.
 * Returns B200_ERR_UNSUPPORTED for shapes outside the envelope (callers fall back to b200_msda_i8). */
int b200_msda_set_i8_resident_bytes(int bytes); /* returns the previous setting */
size_t b200_msda_i8_workspace_size(int batch, int spatial_size, int num_heads, int channels, int num_levels, int num_point,
                                   int points_per_group); /* 0 = shape outside the envelope */
int b200_msda_i8_ws(const int8_t *value, float scale_value, const int32_t *spatial_shapes,
                    const void *reference_points, int ref_is_half, const int8_t *sampling_offsets, float scale_offset,
                    const int8_t *attn_weight, float scale_weight, int batch, int spatial_size, int num_heads,
                    int channels, int num_levels, int num_query, int num_point, int points_per_group, int8_t *out,
                    float scale_out, void *workspace, size_t workspace_bytes, int32_t *trace_records, void *stream);

/* Multi-GPU SCA (SURVEY.md §8(e); not in the reference, which runs spatial_cross_attention.py:270's camera sum on one
 * GPU): reduce-scatter of the fp32 BEV accumulator inside a camera group, over NVLink PEER MEMORY — no NCCL call.
 * The `group_size` ranks of a camera group hold partial sums partials[r][rows*width] (their own cameras only, written
 * by b200_msda_sca_*) for the same query tile; this rank owns floats [first_elem, first_elem + num_elems) of the tile.
 * The kernel (1) publishes step `epoch` into every peer's flag row flags[r][my_index] (release, system scope) and waits
 * until flags[my_index][r] >= epoch for all peers (acquire) — stream order guarantees the local partial is final when
 * the kernel starts; (2) out[i] = sum_r partials[r][first_elem + i], peers read directly over NVLink; (3) zero-fills
 * `zero_next` (the local partial buffer of the NEXT step; partials are double-buffered by step parity).
 *   partials / flags: HOST arrays of `group_size` DEVICE pointers (peer-mapped: torch symmetric memory / cudaIpc);
 *   flags[r] is uint32[10], zero-initialised; epoch starts at 1 and increases by 1 per step on every rank;
 *   out: float (out_is_half == 0) or __half [num_elems]; element counts are multiples of 4.
 * Alignment, for this entry and the three below: partials, out, staging and zero_next are 16-byte aligned (they are
 * moved as float4), every flag row is 4-byte aligned. Any other pointer returns B200_ERR_BAD_PARAM before a launch. */
int b200_sca_peer_reduce(const void *const *partials, void *const *flags, int group_size, int my_index,
                         unsigned int epoch, long long first_elem, long long num_elems, void *out, int out_is_half,
                         float *zero_next, long long zero_elems, void *stream);
/* The same kernel with the step number kept ON THE DEVICE (flags[my_index][8] counts completed steps; the last block of
 * a launch advances it), so that every step's launch has identical parameters and the whole step — sampling launch +
 * this launch — can be captured once into a CUDA graph and replayed. Step s (1, 2, ...) reduces partials_even when
 * s is odd and partials_odd when s is even (the buffers alternate), and zero-fills the OTHER local buffer (zero_elems
 * floats; 0 = do not zero). flags[r] is uint32[10], zero-initialised. */
int b200_sca_peer_reduce_auto(const void *const *partials_even, const void *const *partials_odd, void *const *flags,
                              int group_size, int my_index, long long first_elem, long long num_elems, void *out,
                              int out_is_half, long long zero_elems, void *stream);
/* The overlapped form of the same exchange: a rank first samples the tile rows its PEERS own (launch 1), then its own rows
 * (launch 2). b200_sca_peer_pull_auto — on a side stream, ordered after launch 1 — publishes the step, waits for the
 * peers and pulls THEIR launch-1 results for this rank's slice into `staging` (floats [num_elems], local memory) while
 * launch 2 runs; b200_sca_peer_add_auto — on the main stream after launch 2 and after the pull — writes
 * out = own partial + staging and zero-fills the next step's buffer. Buffers, flags and the device-side step counter are
 * those of b200_sca_peer_reduce_auto, and so are the alignment rules: partial_even / partial_odd, staging and out are
 * 16-byte aligned, flags_local 4-byte aligned. */
int b200_sca_peer_pull_auto(const void *const *partials_even, const void *const *partials_odd, void *const *flags,
                            int group_size, int my_index, long long first_elem, long long num_elems, float *staging,
                            void *stream);
int b200_sca_peer_add_auto(const void *partial_even, const void *partial_odd, void *flags_local, int my_index,
                           long long first_elem, long long num_elems, const float *staging, void *out, int out_is_half,
                           long long zero_elems, void *stream);



/* Trace entries: b200_msda_f32 / _f16 / _i8 with the production kernel's trace switch on (the same kernel template,
 * compiled with one extra store): besides `out` they write, for every (batch, query, head, level*point), the
 * sampling-index record {in_range, h_low, w_low, tap_mask} (4 x int32; all-zero when the point is out of range) that
 * THE GATHER KERNEL ITSELF computed on its way to the taps. Each entry selects its kernel as its plugin op does, except
 * that a traced FP16 launch always uses the exact arithmetic (b200_msda_set_f16_mode 0). `records` must hold
 * batch*num_query*num_heads*num_levels*num_point*4 int32; it is zero-filled on `stream` first. These are what the
 * bit-exact index parity tests compare with the oracle (reference arithmetic: …Kernel.cu:657-674, :138-172). */
int b200_msda_f32_trace(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                        const float *sampling_offsets, const float *attn_weight, int batch, int spatial_size,
                        int num_heads, int channels, int num_levels, int num_query, int num_point,
                        int points_per_group, float *out, int32_t *records, void *stream);
int b200_msda_f16_trace(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                        const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                        int num_heads, int channels, int num_levels, int num_query, int num_point,
                        int points_per_group, void *out, int32_t *records, void *stream);
int b200_msda_bf16_trace(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                         const void *sampling_offsets, const void *attn_weight, int batch, int spatial_size,
                         int num_heads, int channels, int num_levels, int num_query, int num_point,
                         int points_per_group, void *out, int32_t *records, void *stream);
int b200_msda_i8_trace(const int8_t *value, float scale_value, const int32_t *spatial_shapes,
                       const void *reference_points, int ref_is_half, const int8_t *sampling_offsets,
                       float scale_offset, const int8_t *attn_weight, float scale_weight, int batch, int spatial_size,
                       int num_heads, int channels, int num_levels, int num_query, int num_point, int points_per_group,
                       int8_t *out, float scale_out, int32_t *records, void *stream);

/* Stand-alone diagnostic: the same records from a small index-only kernel (no value / logits needed; shares the
 * point_record() device function with the generic fallback kernel). dtype: 0 = float inputs, 1 = __half inputs. */
int b200_msda_debug_indices(int dtype, const int32_t *spatial_shapes, const void *reference_points,
                            const void *sampling_offsets, int batch, int num_heads, int num_levels, int num_query,
                            int num_point, int points_per_group, int32_t *records, void *stream);

/* Backward of b200_msda_f32 / b200_msda_f16 (what mmcv's ms_deform_attn_backward is to the reference's training graph,
 * plus the derivatives of the softmax and of ref * size + offset, which this op computes inside). Same tensors and the
 * same eight ints as the forward, plus grad_output [batch, num_query, num_heads, channels]; each gradient has the layout
 * and dtype of its tensor: grad_value like value, grad_reference_points [batch, num_query, 1, 2 * points_per_group],
 * grad_sampling_offsets like sampling_offsets (pixels), grad_attn_weight like attn_weight (PRE-softmax logits).
 *   - A NULL gradient pointer means that gradient is not computed; requested gradients are OVERWRITTEN.
 *   - Sampling positions follow the forward bit for bit; a point outside the range gate gives zero gradients (it
 *     still counts in the softmax denominator), a tap outside the image is never read.
 *   - All sums accumulate in FP32; FP16 gradients are rounded once, at the end.
 *   - grad_sampling_offsets, grad_attn_weight and grad_reference_points are ordered sums: the same bits on every run,
 *     whichever other gradients are requested. grad_value is reduced with float atomics (not bit-reproducible run to
 *     run, as in mmcv).
 *   - workspace: b200_msda_backward_workspace_size(...) bytes, 256-byte aligned: for FP16 the FP32 accumulator of
 *     grad_value (batch * spatial_size * num_heads * channels * 4 bytes, rounded up to 256), then for both dtypes the
 *     FP32 partials of grad_reference_points (batch * num_query * num_heads * points_per_group * 8 bytes, rounded up
 *     to 256). The query returns 0 for dimensions the entries reject.
 *   - B200_ERR_BAD_PARAM before any launch for a null required pointer (the workspace included), a non-positive
 *     dimension, the forward's size limit ((spatial_size + 1) * num_heads * channels * 4 < 2^31), a pointer that is not
 *     aligned to its element; B200_ERR_UNSUPPORTED for more than 16 levels.
 *   - No host synchronisation and no allocation: the call can be captured in a CUDA graph.
 * Kernels: csrc/msda_backward.cu. channels == 32 with num_point % 4 == 0, points_per_group in {1, 2, 4},
 * num_levels * num_point <= 64 and 16-byte aligned tensors runs the lane-group kernel; every other shape the forward
 * accepts runs a one-thread-per-item kernel. There is no INT8 backward. */
size_t b200_msda_backward_workspace_size(int dtype /* 0 f32, 1 f16, 7 bf16 */, int batch, int spatial_size, int num_heads,
                                         int channels, int num_levels, int num_query, int num_point,
                                         int points_per_group);
int b200_msda_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                           const float *sampling_offsets, const float *attn_weight, const float *grad_output,
                           float *grad_value, float *grad_reference_points, float *grad_sampling_offsets,
                           float *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                           int channels, int num_levels, int num_query, int num_point, int points_per_group,
                           void *stream);
int b200_msda_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                           const void *sampling_offsets, const void *attn_weight, const void *grad_output,
                           void *grad_value, void *grad_reference_points, void *grad_sampling_offsets,
                           void *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                           int channels, int num_levels, int num_query, int num_point, int points_per_group,
                           void *stream);
/* BF16 (b200_msda_bf16): value, offsets, logits, grad_output and their gradients are __nv_bfloat16, reference_points and
 * grad_reference_points FP32. As FP16: FP32 accumulation (grad_value in the workspace), one rounding per gradient.
 * Workspace: b200_msda_backward_workspace_size(7, ...) — the dtype codes follow nvinfer1::DataType (7 = kBF16; 2 is
 * kINT8, which has no backward and keeps returning 0) — the FP16 size. */
int b200_msda_backward_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                            const void *sampling_offsets, const void *attn_weight, const void *grad_output,
                            void *grad_value, float *grad_reference_points, void *grad_sampling_offsets,
                            void *grad_attn_weight, void *workspace, int batch, int spatial_size, int num_heads,
                            int channels, int num_levels, int num_query, int num_point, int points_per_group,
                            void *stream);

/* Backward of the fused SCA forms b200_msda_sca_* (camera-summed) and b200_msda_sca_shared_* (camera-shared), with the
 * conventions of b200_msda_backward_* (NULL gradient = not computed, requested gradients overwritten, argument errors
 * before any launch, no allocation or synchronisation, ordered-sum gradients bit-reproducible) and its workspace query:
 * b200_msda_backward_workspace_size(...) with the same eight ints serves all four entries.
 *   - bev_mask: float [batch, num_query]; grad_slots: float [num_query, num_heads * channels] (the gradient of accum /
 *     slots), both dtypes. The other tensors and gradients have the layout and dtype of the forward's tensors; for the
 *     shared form sampling_offsets / attn_weight and their gradients are the single copy [num_query, ...].
 *   - A (camera, query) pair with bev_mask == 0 contributes nothing to the forward, whatever it samples: it reads
 *     nothing here, adds nothing to grad_value, and gets exact zeros in grad_reference_points and (camera-summed form)
 *     in its offset and logit gradients. Camera-shared form: grad = sum over the cameras with bev_mask != 0, in camera
 *     order; a query no such camera sees gets zero offset and logit gradients.
 *   - B200_ERR_BAD_PARAM as b200_msda_backward_* (bev_mask and grad_slots are required and 4-byte aligned);
 *     B200_ERR_UNSUPPORTED, before any launch, for shapes outside the lane-group kernel: channels != 32,
 *     num_point % 4 != 0, points_per_group not in {1, 2, 4}, num_levels * num_point > 64, or a tensor (grad_slots
 *     included) that is not 16-byte aligned. The forward's fused envelope lies inside it. */
int b200_msda_sca_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                               const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                               const float *grad_slots, float *grad_value, float *grad_reference_points,
                               float *grad_sampling_offsets, float *grad_attn_weight, void *workspace, int batch,
                               int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                               int num_point, int points_per_group, void *stream);
int b200_msda_sca_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                               const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                               const float *grad_slots, void *grad_value, void *grad_reference_points,
                               void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                               int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                               int num_point, int points_per_group, void *stream);
int b200_msda_sca_shared_backward_f32(const float *value, const int32_t *spatial_shapes, const float *reference_points,
                                      const float *sampling_offsets, const float *attn_weight, const float *bev_mask,
                                      const float *grad_slots, float *grad_value, float *grad_reference_points,
                                      float *grad_sampling_offsets, float *grad_attn_weight, void *workspace,
                                      int batch, int spatial_size, int num_heads, int channels, int num_levels,
                                      int num_query, int num_point, int points_per_group, void *stream);
int b200_msda_sca_shared_backward_f16(const void *value, const int32_t *spatial_shapes, const void *reference_points,
                                      const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                                      const float *grad_slots, void *grad_value, void *grad_reference_points,
                                      void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                                      int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                                      int num_point, int points_per_group, void *stream);
/* BF16 forms: dtypes as in b200_msda_backward_bf16 (FP32 reference points and their gradient). */
int b200_msda_sca_backward_bf16(const void *value, const int32_t *spatial_shapes, const float *reference_points,
                                const void *sampling_offsets, const void *attn_weight, const float *bev_mask,
                                const float *grad_slots, void *grad_value, float *grad_reference_points,
                                void *grad_sampling_offsets, void *grad_attn_weight, void *workspace, int batch,
                                int spatial_size, int num_heads, int channels, int num_levels, int num_query,
                                int num_point, int points_per_group, void *stream);
int b200_msda_sca_shared_backward_bf16(const void *value, const int32_t *spatial_shapes,
                                       const float *reference_points, const void *sampling_offsets,
                                       const void *attn_weight, const float *bev_mask, const float *grad_slots,
                                       void *grad_value, float *grad_reference_points, void *grad_sampling_offsets,
                                       void *grad_attn_weight, void *workspace, int batch, int spatial_size,
                                       int num_heads, int channels, int num_levels, int num_query, int num_point,
                                       int points_per_group, void *stream);

/* Selects the FP16 accumulate flavour for b200_msda_f16*. 0 (default) = exact: taps widened to FP32, FP32 weights,
 * packed FP32 FMA (FFMA2) — meets the 1e-3 max-abs parity bar everywhere. 1 = mixed: FP16 tap x FP16 weight -> FP32
 * accumulator (fma.rn.f32.f16, FHFMA); ~15 % fewer issue slots but the FP16 rounding of the weights adds up to ~3e-4
 * on O(1) outputs, so it is opt-in. Returns the previous setting. */
int b200_msda_set_f16_mode(int mode);

/* Selects the kernel behind b200_msda_f16 / _f16_h2 / _f16_trace. 0 (default) = the gather kernel (csrc/msda.cu) for
 * every shape; 1 = the resident-tail kernel (csrc/msda_res.cu: CTAs bound to one (batch, head), the coarsest pyramid
 * levels staged in shared memory by TMA, taps of those levels served from shared memory) whenever channels == 32,
 * num_levels*num_point <= 32, num_point % 4 == 0, and the exact mode of b200_msda_set_f16_mode is selected — measured
 * slower on B200 (DESIGN.md §4.1c), hence opt-in. Same results either way (same index arithmetic, FP32 accumulation).
 * b200_msda_set_resident_bytes: shared memory the resident kernel may use for the tail (default 128 KiB). Both return
 * the previous setting. */
int b200_msda_set_f16_path(int path);
int b200_msda_set_resident_bytes(int bytes);

/* Launch shape of the FP32 / FP16 plugin op (b200_msda_f32 / _f16 / _f16_h2 and their _trace twins): units = 1 is one
 * block of items per CTA; 2 or 4 is the batched launch — every warp first scans the visibility of `units` of its item
 * groups with all their offset / reference-point loads in flight together, answers the invisible ones with zeros and
 * runs the sampling body on the rest (csrc/msda.cu, UPW). strided = 0: the units of a CTA are neighbouring blocks of
 * items; 1: they lie a whole grid apart (evens out CTA run times when visibility comes in long runs). Results are
 * bit-identical for every setting. Any other `units` (e.g. 0) only queries. The initial value is the environment
 * variable B200_MSDA_BATCH ("1", "2", "4", "2s", "4s") if set, else the library default. Returns the previous setting
 * as units | strided << 8. */
int b200_msda_set_batch_units(int units, int strided);

/* Gather depth of the same plugin op (one-unit grid, untraced launches): 0 (default) = 3 CTAs of 8 warps per SM, the 4 tap
 * loads of one sampling point in flight per warp; 1 = 2 CTAs per SM (128-register budget): the 16 tap loads of a 4-point
 * chunk in flight per warp; 2 = the same with that order written out in the source; 3 = 128-thread CTAs, 5 per SM (20 warps,
 * 96 registers), two points = 8 loads issued together — fewer warps, more loads per warp, for inputs on which the kernel is
 * latency-bound. Same bits for every variant (the FMA order does not change). Any other value (e.g. -1) only queries.
 * Initial value: environment variable B200_MSDA_VARIANT ("0" .. "3"), else 0. Returns the
 * previous setting. A batched launch (units > 1 above) combines with variant 1 (batched scan at 2 CTAs per SM) and takes
 * precedence over variants 2 and 3. The fused forms
 * (b200_msda_sca_* / b200_msda_sca_shared_*) have one alternative: any non-zero variant runs them at 2 CTAs per SM. */
int b200_msda_set_gather_variant(int variant);

/* ------------------------------------------------------------------------------------------------------------
 * Plugin-shaped entry: the argument list of IPluginV2DynamicExt::enqueue
 * (…/multiScaleDeformableAttnPlugin.cpp:71-140) with a POD mirror of nvinfer1::PluginTensorDesc, so a TensorRT
 * plugin shell (csrc/trt_plugin/, compiled only where NvInfer.h exists) or any other host can forward verbatim.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t nbDims;
  int32_t d[8];
} b200_dims; /* layout of nvinfer1::Dims */

typedef struct {
  b200_dims dims;
  int32_t type;   /* nvinfer1::DataType: 0 kFLOAT, 1 kHALF, 2 kINT8, 3 kINT32 */
  int32_t format; /* nvinfer1::TensorFormat: 0 kLINEAR, 1 kCHW2 (fp16x2), 2 kHWC8, 3 kCHW4 (int8x4) */
  float scale;
} b200_tensor_desc; /* layout of nvinfer1::PluginTensorDesc */

/* inputs: value, spatial_shapes, reference_points, sampling_offsets, attn_weight; outputs: out.
 * use_h2 selects the …TRT2 flavour. Returns 0 ok / 1 unsupported dtype, as the reference does. */
int b200_msda_enqueue(const b200_tensor_desc *input_desc, const b200_tensor_desc *output_desc,
                      const void *const *inputs, void *const *outputs, void *workspace, void *stream, int use_h2);

/* getWorkspaceSize mirror: bytes b200_msda_enqueue wants in `workspace` for the second-generation INT8 kernels
 * (0 for FP32 / FP16 and for shapes outside their envelope). enqueue(workspace == NULL) runs the round-1 kernels. */
size_t b200_msda_enqueue_workspace_size(const b200_tensor_desc *input_desc);

/* Mirror of supportsFormatCombination (…Plugin.cpp:148-189): 1 if descriptor `pos` of in_out[0..5] is acceptable. */
int b200_msda_supports_format(int pos, const b200_tensor_desc *in_out, int nb_inputs, int nb_outputs);


/* ------------------------------------------------------------------------------------------------------------
 * Grid sampler (plugins GridSampler2DTRT / GridSampler2DTRT2 / GridSampler3DTRT / GridSampler3DTRT2)
 *
 *   input  [N, C, Hi, Wi]       (5-D: [N, C, Di, Hi, Wi])
 *   grid   [N, 2, Ho, Wo]       channel-first: x plane then y plane (5-D: [N, 3, Do, Ho, Wo]); range [-10, 10]
 *   output [N, C, Ho, Wo]
 *   *_dims: HOST int arrays of length nb_dims (4 or 5), as the reference launchers take them.
 *   interp: 0 bilinear, 1 nearest, 2 bicubic (2-D only);  padding: 0 zeros, 1 border, 2 reflection
 *   (enum order of gridSamplerKernel.h:11-12).
 * Semantics = the reference FP32 kernel (TensorRT/plugin/grid_sampler/gridSamplerKernel.cu:666-795, helpers :82-92,
 * :157-162, :226-247, :342-393), evaluated in FP32 for every storage type.
 * ---------------------------------------------------------------------------------------------------------- */

/* replaces grid_sample<float>   — gridSamplerKernel.h:14-18, .cu:1933-1964 */
/* Opt-in tile kernel for 2-D bilinear sampling: 0 (default) = the generic kernel; 1 / 2 = the source window of an 8 x 32
 * output tile is staged in shared memory by TMA (1: one bulk copy per packet row, 2: one 2-D tensor copy per channel
 * packet), with a per-tile fallback to scattered loads when the window does not fit and a per-call fallback when the
 * layout does not meet TMA's 16-byte rules (input pointer, row pitch). Same results bit for bit; measured equal (mode 2)
 * or slower (mode 1) than the generic kernel at the prev-BEV warp. Returns the previous setting. */
int b200_grid_sample_set_tile_path(int mode);
int b200_grid_sample_f32(float *output, const float *input, const float *grid, const int *output_dims,
                         const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                         int align_corners, void *stream);

/* replaces grid_sample<__half>  — same launcher, T=__half, kLINEAR tensors (gridSamplerPlugin.cpp:171-186) */
int b200_grid_sample_f16(void *output, const void *input, const void *grid, const int *output_dims,
                         const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                         int align_corners, void *stream);

/* replaces grid_sample<__half2> — .cu:1969-2008: tensors in TensorRT kCHW2 format
 * (input/output [N, ceil(C/2), H, W, 2]; the 2-channel grid is one (x, y) __half2 per output pixel). 2-D only. */
int b200_grid_sample_f16_chw2(void *output, const void *input, const void *grid, const int *output_dims,
                              const int *input_dims, const int *grid_dims, int nb_dims, int interp, int padding,
                              int align_corners, void *stream);

/* replaces grid_sample_int8     — gridSamplerKernel.h:20-26, .cu:2010-2043: tensors in kCHW4 format
 * (input/output [N, ceil(C/4), H, W, 4] int8; grid (x, y, pad, pad) int8 per output pixel), per-tensor scales,
 * real = q * scale. In-register dequantisation, FP32 math, one requantisation (T2int8). 2-D only. */
int b200_grid_sample_i8_chw4(int8_t *output, float scale_o, const int8_t *input, float scale_i, const int8_t *grid,
                             float scale_g, const int *output_dims, const int *input_dims, const int *grid_dims,
                             int nb_dims, int interp, int padding, int align_corners, void *stream);

/* ------------------------------------------------------------------------------------------------------------
 * Rotate (plugins RotateTRT / RotateTRT2; det2trt/models/functions/rotate.py:7-124)
 *
 *   input / output [C, H, W]   (input_dims = HOST int[3] {C, H, W}, as the plugin passes inputDesc[0].dims.d)
 *   angle  [1] degrees, counter-clockwise; center [2] = (x, y) in pixels: DEVICE pointers (plugin inputs 1, 2)
 *   interp: 0 bilinear, 1 nearest (RotateInterpolation, TensorRT/plugin/rotate/rotateKernel.h:12); zero padding.
 *
 * Semantics = the reference FP32 kernel (rotateKernel.cu:128-210) — its index arithmetic is reproduced operation for
 * operation (b200_rotate_debug_indices exposes it to the tests). FP16 / INT8 images are converted in registers;
 * matrix, coordinates and blending stay FP32 (the reference computes them in half precision, :213-260, :416-456).
 * ---------------------------------------------------------------------------------------------------------- */
/* replaces rotate<float>        — rotateKernel.h:14-16, .cu:708-719 */
int b200_rotate_f32(float *output, const float *input, const float *angle, const float *center,
                    const int *input_dims, int interp, void *stream);

/* replaces rotate<__half>       — same launcher, T=__half: image, angle and center are __half, kLINEAR */
int b200_rotate_f16(void *output, const void *input, const void *angle, const void *center, const int *input_dims,
                    int interp, void *stream);

/* replaces rotate_h2            — rotateKernel.h:18-20, .cu:721-732: image in kCHW2 ([ceil(C/2), H, W, 2] __half) */
int b200_rotate_f16_h2(void *output, const void *input, const void *angle, const void *center, const int *input_dims,
                       int interp, void *stream);

/* replaces rotate_int8<float|__half> — rotateKernel.h:22-26, .cu:734-748: image in kCHW4 ([ceil(C/4), H, W, 4] int8),
 * per-tensor scales (real = q * scale); angle / center are float (angle_is_half = 0) or __half (1), as
 * rotatePlugin.cpp:101-111 dispatches on inputDesc[1].type. */
int b200_rotate_i8(int8_t *output, float scale_o, const int8_t *input, float scale_i, const void *angle,
                   const void *center, int angle_is_half, const int *input_dims, int interp, void *stream);

/* B200 extension: channels-last image [H, W, C] (input_dims still {C, H, W}). prev_bev is stored [H*W, C] at the call
 * site (det2trt/models/modules/transformer.py:296-304); this entry rotates it in place of permute -> RotateTRT ->
 * permute. dtype 0: float image/angle/center, 1: __half. Needs C % 4 == 0 (fp32) / C % 8 == 0 (fp16) and 16-byte
 * aligned buffers, else B200_ERR_UNSUPPORTED. */
int b200_rotate_hwc(void *output, const void *input, const void *angle, const void *center, int dtype,
                    const int *input_dims, int interp, void *stream);

/* Test hook: source_xy[H*W*2] = (ix, iy), the fractional source pixel of every output pixel, from FP32 angle/center. */
int b200_rotate_debug_indices(const float *angle, const float *center, const int *input_dims, float *source_xy,
                              void *stream);


/* ------------------------------------------------------------------------------------------------------------
 * BEV pillar points -> per-camera reference points and visibility weights (the encoder prologue that feeds spatial
 * cross-attention; eager PyTorch in the reference, ONNX elementwise nodes in its engines — no plugin):
 *   BEVFormerEncoderTRTP.get_reference_points_3d  det2trt/models/modules/encoder.py:168-194
 *   BEVFormerEncoderTRTP.point_sampling_trt        det2trt/models/modules/encoder.py:196-259
 *
 *   reference_points      [1, D, bev_h*bev_w, 3] in [0,1] (what get_reference_points_3d returns), or NULL to generate
 *                         that pillar grid analytically (Z = pc_range[5] - pc_range[2], encoder.py:281-289)
 *   pc_range              HOST double[6] = (x0, y0, z0, x1, y1, z1)
 *   lidar2img             DEVICE float [num_cams, 4, 4]
 *   reference_points_cam  [num_cams, 1, Q, D, 2]  (u, v) normalised by (image_w, image_h) — the MSDA reference_points
 *   bev_mask              [num_cams, Q, 1]        seen / max(sum over cameras of seen, 1e-4)
 *   dtype                 0: float tensors, 1: __half tensors (reference_points in, both outputs; math stays FP32 and
 *                         coordinates of points behind a camera saturate to +-65504 instead of overflowing to inf)
 * num_cams <= 16, num_points_in_pillar <= 8, reference_points_cam 16-byte aligned, else B200_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------------------- */
int b200_bev_point_sampling(const void *reference_points, const double *pc_range, const float *lidar2img,
                            int num_cams, int image_h, int image_w, int bev_h, int bev_w, int num_points_in_pillar,
                            int dtype, void *reference_points_cam, void *bev_mask, void *stream);

/* Test hook, host only: out[num_points_in_pillar] = the pillar heights the analytic grid uses (reference_points = NULL),
 * linspace(0.5, Z - 0.5, D) / Z as torch builds it on the CPU, from the same host code as the launch. */
int b200_bev_point_sampling_pillar_heights(const double *pc_range, int num_points_in_pillar, float *out);

/* ------------------------------------------------------------------------------------------------------------
 * Modulated deformable convolution, DCNv2 (plugins ModulatedDeformableConv2dTRT / …TRT2)
 *
 *   input  [batch, channels, height, width]
 *   weight [channels_out, channels/group, kernel_h, kernel_w]     bias [channels_out] or NULL
 *   offset [batch, deformable_group*2*kernel_h*kernel_w, Ho, Wo]  per tap: dh then dw (mmcv order,
 *                                                                 modulatedDeformableConv2dKernel.cu:297-301)
 *   mask   [batch, deformable_group*kernel_h*kernel_w, Ho, Wo]    already sigmoid-ed
 *   output [batch, channels_out, Ho, Wo],  Ho = (height + 2*pad_h - (dilation_h*(kernel_h-1)+1))/stride_h + 1
 *   workspace: device scratch of b200_dcn_workspace_size(...) bytes (the plugin's getWorkspaceSize,
 *              …Conv2dPlugin.cpp:73-115, should return this instead of its single-image column size).
 *   cublas_handle: the reference's slot (…Conv2dPlugin.cpp:286-290), kept for signature compatibility and IGNORED — no
 *   library GEMM runs on this path (dcn_fused.cu: wgmma implicit GEMM; dcn_generic.cu: fused FP32-pipe implicit GEMM)
 *              to use the library's own handle.
 * Argument order = the reference launcher ModulatedDeformConvForwardCUDAKernel<T> (…Conv2dKernel.h:11-19).
 * FP16 accumulates the GEMM in FP32 (the reference accumulates in FP16, common/cuda_helper.cu:101-110).
 * ---------------------------------------------------------------------------------------------------------- */
size_t b200_dcn_workspace_size(int dtype /* 0 f32, 1 f16, 7 bf16 */, int batch, int channels, int height, int width,
                               int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h,
                               int dilation_w, int dilation_h);

/* FP16 runs as one fused implicit GEMM on the tensor cores (wgmma, csrc/dcn_fused.cu) when groups == deformable_groups == 1,
 * channels % 64 == 0 and channels_out in {128, 256, 512}; otherwise (and for FP32) as the generic fused implicit GEMM on
 * the FP32 pipe (csrc/dcn_generic.cu: any groups / deformable groups / kernel size). No library GEMM on either path.
 * b200_dcn_set_fused(0) forces the second path (A/B measurements), a negative argument only queries; returns the
 * previous setting. */
int b200_dcn_set_fused(int enabled);

/* replaces ModulatedDeformConvForwardCUDAKernel<float> — …Conv2dKernel.cu:695-760 */
int b200_dcn_f32(const float *input, const float *weight, const float *bias, const float *offset, const float *mask,
                 float *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                 int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                 int dilation_h, int group, int deformable_group, int im2col_step, void *cublas_handle, void *stream);

/* Deployment helpers for the fused FP16 path (beyond the reference's launcher set): weights are constants at inference
 * time and feature maps may already be channels-last, so both pre-passes of b200_dcn_f16 can be hoisted out of the call.
 *   b200_dcn_pack_weights_f16: weight [Co, C, kh, kw] -> packed [Co][C/64][kh*kw][64] (same byte size), once per layer.
 *   b200_dcn_f16_ex: flags bit 0 = `input` is NHWC [batch, H, W, channels]; bit 1 = `weight` is already packed.
 *   Fused path only (see b200_dcn_set_fused): returns B200_ERR_UNSUPPORTED for other shapes. */
int b200_dcn_pack_weights_f16(const void *weight, void *packed, int channels_out, int channels, int kernel_h, int kernel_w,
                              void *stream);
int b200_dcn_f16_ex(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                    void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                    int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                    int dilation_h, int group, int deformable_group, int flags, void *stream);

/* Backward of b200_dcn_f32 / b200_dcn_f16 (mmcv's modulated_deform_conv_backward, which the reference binding calls).
 * Same tensors and geometry as the forward, plus grad_output [batch, channels_out, Ho, Wo]; gradients in the layout and
 * dtype of their tensors: grad_input like input, grad_weight [channels_out, channels/group, kernel_h, kernel_w],
 * grad_bias [channels_out], grad_offset like offset, grad_mask like mask.
 *   - A NULL gradient pointer means that gradient is not computed; requested gradients are OVERWRITTEN.
 *   - All sums accumulate in FP32; FP16 gradients are rounded once, at the end.
 *   - grad_input is reduced with float atomics (not bit-reproducible run to run, as in mmcv). grad_weight, grad_bias,
 *     grad_offset and grad_mask use ordered reductions: the same bits on every run, whichever other gradients are
 *     requested.
 *   - workspace: b200_dcn_backward_workspace_size(...) bytes, 256-byte aligned (0 = invalid geometry).
 *   - flags (FP16 only) mean what they mean in b200_dcn_f16_ex: bit 0 = `input` is NHWC, bit 1 = `weight` is packed by
 *     b200_dcn_pack_weights_f16. Honoured only for shapes of the fused path (B200_ERR_UNSUPPORTED otherwise); `input`
 *     and `weight` must then be 16-byte aligned. Other bits set are B200_ERR_BAD_PARAM.
 *   - B200_ERR_BAD_PARAM before any launch for null required pointers, bad geometry, channels % group,
 *     channels_out % group, channels % deformable_group, a misaligned pointer.
 *   - kernel_h * kernel_w <= 75 (the data kernel keeps per-tap accumulators in shared memory): larger kernels return
 *     B200_ERR_UNSUPPORTED, and the workspace query returns 0 for them.
 *   - No host synchronisation and no allocation: the call can be captured in a CUDA graph.
 * Kernels: csrc/dcn_backward.cu, one path on the FP32 pipe for every shape and both dtypes (no tensor-core backward
 * yet; b200_dcn_set_fused does not affect it), no library GEMM. NHWC input and packed weights are read in place, so a
 * caller holding the forward's layouts needs no conversion; on this path the plain layouts are the faster ones (at
 * [6,256,58,100] 3x3 on an H100: data kernel +5 % with packed weights, both kernels +15..40 % with an NHWC input). */
size_t b200_dcn_backward_workspace_size(int dtype /* 0 f32, 1 f16, 7 bf16 */, int batch, int channels, int height, int width,
                                        int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h,
                                        int pad_w, int pad_h, int dilation_w, int dilation_h, int group,
                                        int deformable_group);
int b200_dcn_backward_f32(const float *input, const float *weight, const float *offset, const float *mask,
                          const float *grad_output, float *grad_input, float *grad_weight, float *grad_bias,
                          float *grad_offset, float *grad_mask, void *workspace, int batch, int channels, int height,
                          int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                          int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, void *stream);
int b200_dcn_backward_f16(const void *input, const void *weight, const void *offset, const void *mask,
                          const void *grad_output, void *grad_input, void *grad_weight, void *grad_bias,
                          void *grad_offset, void *grad_mask, void *workspace, int batch, int channels, int height,
                          int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                          int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, int flags,
                          void *stream);
/* BF16: the FP32 entry's arguments (no flags), every tensor and gradient __nv_bfloat16, FP32 accumulation with grad_input
 * in the workspace (b200_dcn_backward_workspace_size(7, ...) = the FP16 size), one rounding per gradient. */
int b200_dcn_backward_bf16(const void *input, const void *weight, const void *offset, const void *mask,
                           const void *grad_output, void *grad_input, void *grad_weight, void *grad_bias,
                           void *grad_offset, void *grad_mask, void *workspace, int batch, int channels, int height,
                           int width, int channels_out, int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w,
                           int pad_h, int dilation_w, int dilation_h, int group, int deformable_group, void *stream);

/* replaces ModulatedDeformConvForwardCUDAKernel_int8<float> / <__half> — …Conv2dKernel.h:21-29, .cu:897-978.
 * input int8 kCHW4 [batch, channels/4, H, W, 4], weight int8 kCHW4 [channels_out, channels/4, kh, kw, 4], offset / mask
 * int8 kLINEAR, output int8 kLINEAR, per-tensor scales (real = q*scale); bias float (bias_is_half == 0), __half, or NULL.
 * Arithmetic: in-register dequantisation (int8 values are exact in FP16), FP16 tensor-core products with FP32
 * accumulation, one requantisation T2int8((acc*scale_i*scale_w + bias)/scale_o) — the reference requantises the
 * sampled columns to int8 first (:536-545). Shapes of the fused path (groups == deformable_groups == 1,
 * channels % 64 == 0, channels_out in {128, 256, 512}) run on tensor cores in one kernel; any other shape with
 * channels % 4 == 0 and (channels / group) % 4 == 0 dequantises into the workspace and runs the generic hand-written FP16
 * kernel (csrc/dcn_generic.cu, FP32 accumulation), one requantisation at the end. workspace: b200_dcn_i8_workspace_size(...) bytes,
 * 256-byte aligned. `input` and `weight` must be 4-byte aligned (their kCHW4 packets are read as 32-bit words); an
 * unaligned pointer returns B200_ERR_UNSUPPORTED before anything is launched. */
size_t b200_dcn_i8_workspace_size(int batch, int channels, int height, int width, int channels_out, int kernel_w,
                                  int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                                  int dilation_h, int group, int deformable_group);
int b200_dcn_i8(const int8_t *input, float scale_i, const int8_t *weight, float scale_w, const void *bias, int bias_is_half,
                const int8_t *offset, float scale_off, const int8_t *mask, float scale_mask, int8_t *output, float scale_o,
                void *workspace, int batch, int channels, int height, int width, int channels_out, int kernel_w,
                int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w, int dilation_h, int group,
                int deformable_group, int im2col_step, void *cublas_handle, void *stream);

/* replaces ModulatedDeformConvForwardCUDAKernel<__half> / <__half2> — …Conv2dKernel.cu:762-895 (kLINEAR tensors) */
int b200_dcn_f16(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                 void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                 int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                 int dilation_h, int group, int deformable_group, int im2col_step, void *cublas_handle, void *stream);

/* BF16 (beyond the reference): every tensor __nv_bfloat16, on the generic kernel (csrc/dcn_generic.cu) for every shape
 * — there is no BF16 tensor-core path. Each element widened to FP32 exactly, FP32 accumulation, one rounding per output.
 * workspace: b200_dcn_workspace_size(7, ...) bytes (dtype codes follow nvinfer1::DataType:
 * 7 = kBF16). */
int b200_dcn_bf16(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                  void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                  int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                  int dilation_h, int group, int deformable_group, int im2col_step, void *cublas_handle, void *stream);

/* FP16 in TensorRT's kCHW2 packets — what the …TRT2 plugin negotiates (…Conv2dPlugin.cpp:222-250: input, offset and
 * weight as __half2 packets [N, ceil(C/2), H, W, 2]; mask, bias and output linear). Replaces
 * ModulatedDeformConvForwardCUDAKernel<__half2> (…Conv2dKernel.cu:828-895). The packets are unpacked into the workspace
 * (sized by b200_dcn_f16_chw2_workspace_size) and the FP16 path above runs. */
size_t b200_dcn_f16_chw2_workspace_size(int batch, int channels, int height, int width, int channels_out, int kernel_w,
                                        int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                                        int dilation_h, int group, int deformable_group);
int b200_dcn_f16_chw2(const void *input, const void *weight, const void *bias, const void *offset, const void *mask,
                      void *output, void *workspace, int batch, int channels, int height, int width, int channels_out,
                      int kernel_w, int kernel_h, int stride_w, int stride_h, int pad_w, int pad_h, int dilation_w,
                      int dilation_h, int group, int deformable_group, int im2col_step, void *cublas_handle, void *stream);

/* ------------------------------------------------------------------------------------------------------------
 * Plugin-shaped entries for the other two plugins (the argument list of IPluginV2DynamicExt::enqueue plus the plugin's
 * attributes), so that a TensorRT shell — or a test — forwards verbatim, as b200_msda_enqueue does for MSDA.
 * ---------------------------------------------------------------------------------------------------------- */
/* GridSampler{2D,3D}TRT[2] (gridSamplerPlugin.cpp:110-155): inputs = input, grid; dispatch on the input descriptor's
 * type / format (fp32, fp16 linear, fp16 kCHW2, int8 kCHW4 with the descriptors' scales). The grid and output
 * descriptors must have the input's rank and the output dims must be [N, C, grid spatial], else B200_ERR_BAD_PARAM.
 * Needs no workspace. */
int b200_grid_sampler_enqueue(const b200_tensor_desc *input_desc, const b200_tensor_desc *output_desc,
                              const void *const *inputs, void *const *outputs, void *workspace, void *stream,
                              int interpolation_mode, int padding_mode, int align_corners);
/* supportsFormatCombination mirror (gridSamplerPlugin.cpp:168-194): in_out = {input, grid, output}. */
int b200_grid_sampler_supports_format(int pos, const b200_tensor_desc *in_out, int nb_inputs, int nb_outputs, int use_h2);

/* RotateTRT[2] (rotatePlugin.cpp:75-113): inputs = img [C, H, W], angle [1], center [2]; interp = the plugin attribute,
 * use_h2 = the …TRT2 flavour (FP16 as kCHW2 packets). B200_ERR_BAD_PARAM unless img has rank 3, the output dims equal
 * img's, angle has 1 element and center 2. Dispatch on img's type: fp32, fp16, int8 kCHW4 with the descriptors' scales
 * (angle / center __half when the angle descriptor is kHALF). Needs no workspace. */
int b200_rotate_enqueue(const b200_tensor_desc *input_desc, const b200_tensor_desc *output_desc,
                        const void *const *inputs, void *const *outputs, void *workspace, void *stream, int interp,
                        int use_h2);
/* supportsFormatCombination mirror (rotatePlugin.cpp:122-153): in_out = {img, angle, center, output}. */
int b200_rotate_supports_format(int pos, const b200_tensor_desc *in_out, int nb_inputs, int nb_outputs, int use_h2);

/* ModulatedDeformableConv2dTRT[2] (…Conv2dPlugin.cpp:117-199): inputs = x, offset, mask, weight[, bias] (nb_inputs 4 or
 * 5). stride / padding / dilation = the plugin attributes' int[2] in ONNX order (h, w), as the exporter writes them
 * (stride_i=_pair(stride)): element [0] is handed to the launcher's *_h slot and [1] to *_w. (The reference's enqueue,
 * :152-160, hands [0] to *_w, so its launch disagrees with its own output dimensions for asymmetric layers.)
 * Before anything is launched, Ho / Wo are computed from the input, weight and attributes, and B200_ERR_BAD_PARAM is
 * returned unless offset = [N, dg*2*kh*kw, Ho, Wo], mask = [N, dg*kh*kw, Ho, Wo], output = [N, Co, Ho, Wo],
 * weight.d1 * groups = C and (with 5 inputs) bias = [Co]. Dispatch: fp32, fp16 linear, fp16 kCHW2, int8 kCHW4. */
size_t b200_dcn_enqueue_workspace_size(const b200_tensor_desc *input_desc, const int32_t *stride, const int32_t *padding,
                                       const int32_t *dilation, int groups, int deform_groups);
int b200_dcn_enqueue(const b200_tensor_desc *input_desc, const b200_tensor_desc *output_desc, const void *const *inputs,
                     void *const *outputs, void *workspace, void *stream, int nb_inputs, const int32_t *stride,
                     const int32_t *padding, const int32_t *dilation, int groups, int deform_groups);
/* supportsFormatCombination mirror (…Conv2dPlugin.cpp:213-250): in_out = {x, offset, mask, weight[, bias], output};
 * groups = the plugin attribute (INT8 needs C and Co / groups to be multiples of 4). */
int b200_dcn_supports_format(int pos, const b200_tensor_desc *in_out, int nb_inputs, int nb_outputs, int groups,
                             int use_h2);

/* ------------------------------------------------------------------------------------------------------------
 * BEVPoolV2 (plugins BEVPoolV2TRT / BEVPoolV2TRT2; TensorRT/plugin/bev_pool_v2/bevPoolKernel.h, backward
 * third_party/bev_mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu) — BEVDet's lift-splat pooling:
 *
 *   depth            [N, D, H, W]      depth_size = N*D*H*W elements
 *   feat             [N, H, W, C]      channels last; feat_rows = N*H*W rows of `channels`
 *   ranks_depth, ranks_feat, ranks_bev   int32 [num_points]
 *   interval_starts, interval_lengths    int32 [num_intervals]
 *   out              [1, out_height, out_width, C]
 *
 *   out[ranks_bev[s_k], c] = sum_{i = s_k}^{s_k + len_k - 1} feat[ranks_feat[i], c] * depth[ranks_depth[i]]
 * with s_k = interval_starts[k], len_k = interval_lengths[k]; every cell no interval names is +0 (filled on `stream`).
 * Contract (what voxel_pooling_prepare_v2 produces): points sorted by ranks_bev, one interval per distinct cell, each
 * depth element referenced by at most one point. Index safety: [s_k, s_k + len_k) is clipped to [0, num_points); an
 * interval whose cell ranks_bev[max(s_k, 0)] is outside [0, out_height*out_width) is dropped, and so is a point whose
 * ranks_depth or ranks_feat is outside its tensor; no input forms an address outside a tensor.
 * Numerics: FP32 = the reference kernel's FFMA chain in point order, bit for bit. FP16 and BF16 accumulate in FP32 and
 * round once. INT8 (channels % 4 == 0, else B200_ERR_UNSUPPORTED): exact int32 sum, one multiply by
 * scale_depth * scale_feat / scale_out (evaluated in float on the host), saturate, round half away from zero.
 * Pointers of zero-length arrays may be NULL; any other NULL pointer, a pointer not aligned to its element (4 bytes
 * for float and int32, 2 for half and bfloat16) or a negative size is B200_ERR_BAD_PARAM.
 *
 * Element types per entry (the `f32_depth` entries take what torch.autocast hands the op: a softmax depth in FP32 and
 * conv features in FP16 / BF16; feat_dtype = 1 for fp16, 7 for bf16, nvinfer1::DataType's codes, and any other value is
 * B200_ERR_UNSUPPORTED before anything is launched):
 *
 *   entry                    depth   feat, out   depth_grad   out_grad, feat_grad
 *   _f32                     fp32    fp32        fp32         fp32
 *   _f16                     fp16    fp16        fp16         fp16
 *   _bf16                    bf16    bf16        bf16         bf16
 *   _f32_depth, feat_dtype 1 fp32    fp16        fp32         fp16
 *   _f32_depth, feat_dtype 7 fp32    bf16        fp32         bf16
 *
 * Every 2-byte element is widened to FP32 exactly and FP32 depth is used as loaded; the forward is the FP32 FFMA chain
 * in point order and each 2-byte result is rounded once, to nearest even. An FP32 depth gradient is not rounded. FP32
 * depth and its gradient must be 4-byte aligned, every 2-byte tensor 2-byte aligned. */
int b200_bev_pool_f32(const float *depth, const float *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                      const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                      int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                      int out_height, int out_width, float *out, void *stream);
int b200_bev_pool_f16(const void *depth, const void *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                      const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                      int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                      int out_height, int out_width, void *out, void *stream);
int b200_bev_pool_bf16(const void *depth, const void *feat, const int32_t *ranks_depth, const int32_t *ranks_feat,
                       const int32_t *ranks_bev, const int32_t *interval_starts, const int32_t *interval_lengths,
                       int channels, int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                       int out_height, int out_width, void *out, void *stream);
int b200_bev_pool_f32_depth(int feat_dtype, const float *depth, const void *feat, const int32_t *ranks_depth,
                            const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                            const int32_t *interval_lengths, int channels, int num_points, int num_intervals,
                            int64_t depth_size, int64_t feat_rows, int out_height, int out_width, void *out,
                            void *stream);
int b200_bev_pool_i8(const int8_t *depth, float scale_depth, const int8_t *feat, float scale_feat,
                     const int32_t *ranks_depth, const int32_t *ranks_feat, const int32_t *ranks_bev,
                     const int32_t *interval_starts, const int32_t *interval_lengths, int channels, int num_points,
                     int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                     int8_t *out, float scale_out, void *stream);

/* Backward of b200_bev_pool_f32 / _f16 / _bf16 / _f32_depth, each gradient in its argument's dtype (the table above)
 * with FP32 accumulation and no atomics (the same bits on every run and for every subset of gradients asked for):
 *   depth_grad[ranks_depth[i]] = sum_c out_grad[cell(i), c] * feat[ranks_feat[i], c]
 *   feat_grad[f, c]            = sum_{i : ranks_feat[i] = f} out_grad[cell(i), c] * depth[ranks_depth[i]]
 * where cell(i) is the cell of the interval that pooled point i (= ranks_bev[i] within the contract); both are zero
 * where no pooled point refers. Either gradient pointer may be NULL (not both). feat_order = the point indices sorted
 * by ranks_feat with equal keys in index order (a stable argsort, the reference backward's regrouping); needed with
 * feat_grad only. workspace: b200_bev_pool_backward_workspace_size(num_points) bytes of device memory. */
size_t b200_bev_pool_backward_workspace_size(int num_points);
int b200_bev_pool_backward_f32(const float *out_grad, const float *depth, const float *feat, const int32_t *ranks_depth,
                               const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                               const int32_t *interval_lengths, const int32_t *feat_order, int channels, int num_points,
                               int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                               float *depth_grad, float *feat_grad, void *workspace, size_t workspace_size,
                               void *stream);
int b200_bev_pool_backward_f16(const void *out_grad, const void *depth, const void *feat, const int32_t *ranks_depth,
                               const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                               const int32_t *interval_lengths, const int32_t *feat_order, int channels, int num_points,
                               int num_intervals, int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                               void *depth_grad, void *feat_grad, void *workspace, size_t workspace_size,
                               void *stream);
int b200_bev_pool_backward_bf16(const void *out_grad, const void *depth, const void *feat, const int32_t *ranks_depth,
                                const int32_t *ranks_feat, const int32_t *ranks_bev, const int32_t *interval_starts,
                                const int32_t *interval_lengths, const int32_t *feat_order, int channels,
                                int num_points, int num_intervals, int64_t depth_size, int64_t feat_rows,
                                int out_height, int out_width, void *depth_grad, void *feat_grad, void *workspace,
                                size_t workspace_size, void *stream);
int b200_bev_pool_backward_f32_depth(int feat_dtype, const void *out_grad, const float *depth, const void *feat,
                                     const int32_t *ranks_depth, const int32_t *ranks_feat, const int32_t *ranks_bev,
                                     const int32_t *interval_starts, const int32_t *interval_lengths,
                                     const int32_t *feat_order, int channels, int num_points, int num_intervals,
                                     int64_t depth_size, int64_t feat_rows, int out_height, int out_width,
                                     float *depth_grad, void *feat_grad, void *workspace, size_t workspace_size,
                                     void *stream);

/* BEVPoolV2TRT[2] (bevPoolPlugin.cpp:71-117): inputs = depth, feat, ranks_depth, ranks_feat, ranks_bev,
 * interval_starts, interval_lengths; output [1, out_height, out_width, C]. Extents come from the descriptors, which
 * must agree (index arrays 1-D of matching lengths, output dims = {1, out_height, out_width, feat's last dim}), else
 * B200_ERR_BAD_PARAM. Dispatch on the depth descriptor's type: fp32, fp16 or int8 (scales from the descriptors). Both
 * plugin names run the same kernels. Needs no workspace. */
int b200_bev_pool_enqueue(const b200_tensor_desc *input_desc, const b200_tensor_desc *output_desc,
                          const void *const *inputs, void *const *outputs, void *workspace, void *stream,
                          int out_height, int out_width);
/* supportsFormatCombination mirror: in_out = {the seven inputs, output}; positions 0, 1 and 7 fp32, fp16 or int8
 * (int8 when C % 4 == 0) kLINEAR of one type, positions 2-6 int32 kLINEAR. */
int b200_bev_pool_supports_format(int pos, const b200_tensor_desc *in_out, int nb_inputs, int nb_outputs);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* B200_BEV_OPS_H */
