/*
 * fn2b200.h -- C ABI of libfn2b200.so: H100 (sm_90a) kernels for flownet2-pytorch's three
 * custom layers.  This is the drop-in boundary: plain pointers and sizes, no torch types.
 *
 * Each entry point replaces one function of the reference's pybind extensions
 * (paths relative to the reference's networks/ directory):
 *
 *   fn2b200_correlation_forward    <- correlation_package/correlation_cuda.cc:10-87
 *                                     (+ correlation_cuda_kernel.cu:336-427: K1 x2, K2)
 *   fn2b200_correlation_backward   <- correlation_package/correlation_cuda.cc:89-167
 *                                     (+ correlation_cuda_kernel.cu:430-564: K1 x2, K3 xB, K4 xB)
 *   fn2b200_correlation_out_shape  <- correlation_package/correlation_cuda.cc:19-34
 *   fn2b200_resample2d_forward     <- resample2d_package/resample2d_cuda.cc:6-13
 *                                     (+ resample2d_kernel.cu:200-242: K5)
 *   fn2b200_resample2d_backward    <- resample2d_package/resample2d_cuda.cc:15-24
 *                                     (+ resample2d_kernel.cu:244-323: K6, K7)
 *   fn2b200_channelnorm_forward    <- channelnorm_package/channelnorm_cuda.cc:6-13
 *                                     (+ channelnorm_kernel.cu:98-129: K8)
 *   fn2b200_channelnorm_backward   <- channelnorm_package/channelnorm_cuda.cc:16-25
 *                                     (+ channelnorm_kernel.cu:131-177: K9)
 *
 * Conventions
 *   - All data pointers are DEVICE pointers to fp32.  The device need not be current: every call
 *     binds the calling thread to the device that owns its first data pointer
 *     (cudaPointerGetAttributes + cudaSetDevice), so autograd worker threads and nn.DataParallel
 *     replica threads can call in without a context.  Tensors are contiguous NCHW unless a stride
 *     array is passed.
 *   - `stream` is a cudaStream_t / CUstream handle (NULL = legacy default stream).  Calls are
 *     asynchronous with respect to the host, like the reference (it never synchronises).
 *   - Return value: 0 on success; a negative FN2B200_E* code for argument errors; a positive
 *     cudaError_t value when the CUDA runtime reported a failure.  fn2b200_last_error() returns a
 *     thread-local human-readable message for the last failing call on this thread.  (The
 *     reference raises AT_ERROR("CUDA call failed"), correlation_cuda.cc:81-83; the Python host
 *     layer turns a non-zero return into RuntimeError.)
 *   - The library keeps no mutable global state (bar a launch counter): every call is re-entrant and thread-safe
 *     (nn.DataParallel calls these from one Python thread per GPU, main.py:200).
 *   - Outputs are fully overwritten; no pre-zeroing is required except where noted.
 *   - No entry point synchronises, allocates device memory or keeps state between calls (scratch is always a
 *     caller-provided workspace; fills are cudaMemsetAsync on `stream`), so every call can be captured into a CUDA
 *     graph on a capturing stream.
 */
#ifndef FN2B200_H_
#define FN2B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FN2B200_VERSION 100

#define FN2B200_EINVAL (-1)      /* bad shape / parameter */
#define FN2B200_EUNSUPPORTED (-2) /* parameter combination the reference itself cannot run */
#define FN2B200_ENULL (-3)       /* null pointer with a non-empty tensor */

int fn2b200_version(void);
const char *fn2b200_last_error(void);

/* D = (2*(md/s2)+1)^2, oH/oW = ceil((H + 2*pad - 2*((k-1)/2 + md)) / s1)  (float ceil). */
int fn2b200_correlation_out_shape(int C, int H, int W, int pad_size, int kernel_size,
                                  int max_displacement, int stride1, int stride2, int *D,
                                  int *oH, int *oW);

/*
 * fn2b200_correlation_forward_cat with cat_channels = D, ch_offset = 0, leaky_slope = 1 and no workspace (FP32-FMA
 * kernels): output [B,D,oH,oW].  No padded/transposed scratch tensors are needed (the reference's rInput1/rInput2 have
 * no counterpart here).
 */
int fn2b200_correlation_forward(const float *input1, const float *input2, float *output, int B,
                                int C, int H, int W, int pad_size, int kernel_size,
                                int max_displacement, int stride1, int stride2,
                                int corr_type_multiply, void *stream);

/*
 * fn2b200_correlation_forward_workspace() returns the workspace bytes of the tensor-core forward (0 = the FP32-FMA
 * kernels run: configuration not supported, or FN2B200_CORR_FWD=fma).  fn2b200_correlation_forward_ws() equals
 * fn2b200_correlation_forward_cat with cat_channels = D, ch_offset = 0, leaky_slope = 1: output [B,D,oH,oW].
 */
size_t fn2b200_correlation_forward_workspace(int B, int C, int H, int W, int pad_size, int kernel_size,
                                             int max_displacement, int stride1, int stride2);
int fn2b200_correlation_forward_ws(const float *input1, const float *input2, float *output, int B, int C,
                                   int H, int W, int pad_size, int kernel_size, int max_displacement,
                                   int stride1, int stride2, int corr_type_multiply, void *workspace,
                                   size_t workspace_bytes, void *stream);

/*
 * The correlation forward.  input1, input2: [B,C,H,W]; cat: [B, cat_channels, oH, oW].  Writes
 * LeakyReLU(leaky_slope)(correlation) into channels [ch_offset, ch_offset + D) of cat and leaves its other channels
 * untouched; leaky_slope = 1 writes the plain correlation.  SURVEY 8(f)-2 (FlowNetC.py:86-92): FlowNetC's 473-channel
 * concat holds conv_redir's 32 channels first, then the 441 displacement channels, so neither the activation's
 * read-modify-write nor torch.cat's copy of the cost volume happens.
 * Tensor cores (wgmma, bf16 hi/lo operand split, fp32 accumulation in registers; error ~1e-5 relative, inside the 1e-4
 * contract) run when the configuration supports them and the workspace holds at least
 * fn2b200_correlation_forward_workspace() bytes; it must then be 128-byte aligned (else FN2B200_EINVAL).  A NULL or
 * smaller workspace, or FN2B200_CORR_FWD=fma, selects the FP32-FMA kernels.  The workspace plays the role of the
 * reference's rInput1/rInput2 scratch tensors (correlation_cuda.cc:36-41) and may be reused or freed (stream-ordered)
 * as soon as the call returns.  corr_type_multiply is accepted and ignored, exactly as in the reference
 * (correlation_cuda_kernel.cu:369).
 * Bad shape or parameters, an empty output, a channel range outside the buffer or a tensor of 2^31 elements or more ->
 * FN2B200_EINVAL; NULL input1, input2 or cat -> FN2B200_ENULL; B == 0 is a no-op.  Its backward is
 * fn2b200_correlation_backward_cat.
 */
int fn2b200_correlation_forward_cat(const float *input1, const float *input2, float *cat, int cat_channels,
                                    int ch_offset, float leaky_slope, int B, int C, int H, int W, int pad_size,
                                    int kernel_size, int max_displacement, int stride1, int stride2,
                                    int corr_type_multiply, void *workspace, size_t workspace_bytes, void *stream);

/*
 * fn2b200_correlation_backward_workspace() returns the workspace bytes of the tensor-core backward (same size and
 * layout as the forward's; 0 = FP32-FMA kernels, also under FN2B200_CORR_BWD=fma).  fn2b200_correlation_backward_ws()
 * equals fn2b200_correlation_backward_cat with cat_channels = D, ch_offset = 0, leaky_slope = 1 (cat unused):
 * grad_output [B,D,oH,oW].
 */
size_t fn2b200_correlation_backward_workspace(int B, int C, int H, int W, int pad_size, int kernel_size,
                                              int max_displacement, int stride1, int stride2);
int fn2b200_correlation_backward_ws(const float *input1, const float *input2, const float *grad_output,
                                    float *grad_input1, float *grad_input2, int B, int C, int H, int W,
                                    int pad_size, int kernel_size, int max_displacement, int stride1,
                                    int stride2, int corr_type_multiply, void *workspace,
                                    size_t workspace_bytes, int workspace_has_split, void *stream);

/*
 * The correlation backward: the input gradients of
 *     cat[:, ch_offset : ch_offset + D] = LeakyReLU(leaky_slope)(correlation(input1, input2))
 * given grad_cat, the gradient of the whole [B, cat_channels, oH, oW] concat buffer, and `cat`, the buffer the forward
 * wrote (same layout; only its [ch_offset, ch_offset + D) channels are read).  Every gradOutput value is
 *     gO[n,d,p] = grad_cat[n, ch_offset+d, p] * (cat[n, ch_offset+d, p] > 0 ? 1 : leaky_slope)
 * (LeakyReLU's derivative read from its output, as torch's in-place LeakyReLU does), applied per element before any
 * other arithmetic, so the result is bit-identical to the plain backward on that masked, dense gO.  The slice is read in
 * place: no masked copy of the cost volume is written, and the tensor-core path stays one launch.  leaky_slope = 1: no
 * activation (cat may be NULL).  grad_input1, grad_input2: [B,C,H,W]; either may be NULL to skip it (both NULL: no-op).
 * Workspace as in fn2b200_correlation_forward_cat (FN2B200_CORR_BWD=fma forces the FP32-FMA kernels);
 * workspace_has_split != 0 promises that it still holds what the forward wrote for the SAME input1/input2 (the split
 * pass is then skipped).
 * leaky_slope < 0 (the output's sign no longer gives the mask), bad shape or parameters, a channel range outside the
 * buffer or a tensor of 2^31 elements or more -> FN2B200_EINVAL; stride1 != 1 -> FN2B200_EUNSUPPORTED (the reference's
 * backward indexes out of bounds, correlation_cuda_kernel.cu:163-164 vs :520); NULL input1, input2, grad_cat, or cat
 * with leaky_slope != 1 -> FN2B200_ENULL; B == 0 is a no-op.
 */
int fn2b200_correlation_backward_cat(const float *input1, const float *input2, const float *grad_cat, const float *cat,
                                     int cat_channels, int ch_offset, float leaky_slope, float *grad_input1,
                                     float *grad_input2, int B, int C, int H, int W, int pad_size, int kernel_size,
                                     int max_displacement, int stride1, int stride2, int corr_type_multiply,
                                     void *workspace, size_t workspace_bytes, int workspace_has_split, void *stream);

/*
 * fn2b200_correlation_backward_cat with cat_channels = D, ch_offset = 0, leaky_slope = 1 and no workspace (FP32-FMA
 * kernels): grad_output [B,D,oH,oW].
 */
int fn2b200_correlation_backward(const float *input1, const float *input2,
                                 const float *grad_output, float *grad_input1,
                                 float *grad_input2, int B, int C, int H, int W, int pad_size,
                                 int kernel_size, int max_displacement, int stride1, int stride2,
                                 int corr_type_multiply, void *stream);

/*
 * input1 (image): [*,C,iH,iW] with element strides istride[4] = {b, c, h, w} (so the
 * non-contiguous channel slice models.py:133 passes needs no .contiguous() copy);
 * input2 (flow): [B,2,H,W] contiguous; output: [B,C,H,W] contiguous.
 * kernel_size must be 1 (the reference's kernel_size > 1 taps are unclamped and read out of
 * bounds, resample2d_kernel.cu:54-61) -> FN2B200_EUNSUPPORTED.  bilinear == 0 -> nearest.
 */
int fn2b200_resample2d_forward(const float *input1, const int64_t *istride, const float *input2,
                               float *output, int B, int C, int iH, int iW, int H, int W,
                               int kernel_size, int bilinear, void *stream);

/*
 * grad_output: [B,C,H,W]; grad_input1: [B,C,iH,iW] contiguous; grad_input2: [B,2,H,W].
 * grad_input1 is accumulated with fp32 atomics (order non-deterministic, like the reference's
 * atomicAdd, resample2d_kernel.cu:118-121).  zero_grad_input1 != 0 -> the library zero-fills it
 * on `stream` first; 0 -> the caller already did (resample2d.py:31).  Either grad may be NULL.
 * The backward is always the bilinear one (`bilinear` is ignored, as in the reference).
 */
int fn2b200_resample2d_backward(const float *input1, const int64_t *istride, const float *input2,
                                const float *grad_output, float *grad_input1, float *grad_input2,
                                int B, int C, int iH, int iW, int H, int W, int kernel_size,
                                int bilinear, int zero_grad_input1, void *stream);

/*
 * Backward with a caller-provided scratch: fn2b200_resample2d_backward_workspace() returns the bytes needed (0 = C > 3:
 * scalar reductions straight into grad_input1, what fn2b200_resample2d_backward does), and
 * fn2b200_resample2d_backward_ws() is fn2b200_resample2d_backward() plus a 16-byte aligned device workspace of at least
 * that size (NULL is fine when grad_input1 is NULL).  The image gradient is accumulated in the workspace as ONE
 * 16-byte vector reduction per bilinear tap (pixel-interleaved layout [B][iH][iW][4]: 4 lane-operations per pixel
 * instead of 4 C) and transposed into grad_input1 afterwards: grad_input1 then needs no zero fill; with
 * zero_grad_input1 == 0 the result is ADDED to what it holds.
 */
size_t fn2b200_resample2d_backward_workspace(const int64_t *istride, int B, int C, int iH, int iW, int H, int W);
int fn2b200_resample2d_backward_ws(const float *input1, const int64_t *istride, const float *input2,
                                   const float *grad_output, float *grad_input1, float *grad_input2, int B, int C,
                                   int iH, int iW, int H, int W, int kernel_size, int bilinear, int zero_grad_input1,
                                   void *workspace, size_t workspace_bytes, void *stream);

/*
 * SURVEY 8(f)-3: Resample2d whose flow is still at quarter resolution.  output = Resample2d()(input1, up(flow * flow_mul))
 * where up = nn.Upsample(scale_factor=4, mode='bilinear') (upsample_mode 1; align_corners=False arithmetic) or
 * mode='nearest' (upsample_mode 2) -- the chain the reference spells out at models.py:130-133, :142-145, :154-157,
 * :167-168 -- without the full-resolution flow ever being written.  flow: [B,2,fh,fw] contiguous with H = 4 fh,
 * W = 4 fw (upsample_mode 0: fh = H, fw = W, flow_mul ignored).  input1 as in fn2b200_resample2d_forward (any
 * element strides, any C) with iH = H, iW = W.
 */
int fn2b200_resample2d_forward_up(const float *input1, const int64_t *istride, const float *flow, int fh, int fw,
                                  int upsample_mode, float flow_mul, float *output, int B, int C, int H, int W,
                                  void *stream);

/*
 * SURVEY 8(f)-1: warp -> diff -> channel-norm -> concat in one kernel (models.py:133-138, :145-150, :155-161, :168-174).
 * x: [B, >= 2C, H, W] with element strides xstride[4] (unit stride along W), img0 = x[:, :C], img1 = x[:, C:2C].
 * flow / fh / fw / upsample_mode / flow_mul: as in fn2b200_resample2d_forward_up (flow_up below is the upsampled flow).
 * cat: [B, cat_channels, H, W] contiguous; each ch_* names the first channel of one product, negative = not wanted:
 *   ch_x         n_x channels      x[:, :n_x]                                  (n_x <= 2C)
 *   ch_warped    C channels        warped = Resample2d()(img1, flow_up)
 *   ch_flow      2 channels        flow_up / flow_div
 *   ch_flow_norm 1 channel         ChannelNorm()(flow_up)
 *   ch_diff_norm 1 channel         ChannelNorm()(img0 - warped)
 * Channel ranges must not overlap; channels no product covers are left untouched.  models.py:138's concat1 is {cat_channels 12, ch_x 0, n_x 6, ch_warped 6, ch_flow 9,
 * flow_div = div_flow, ch_flow_norm -1, ch_diff_norm 11}.
 */
int fn2b200_warp_concat_forward(const float *x, const int64_t *xstride, int C, const float *flow, int fh, int fw,
                                int upsample_mode, float flow_mul, float *cat, int cat_channels, int ch_x, int n_x,
                                int ch_warped, int ch_flow, float flow_div, int ch_flow_norm, int ch_diff_norm, int B,
                                int H, int W, void *stream);

/*
 * Backward of fn2b200_warp_concat_forward, C <= 3, flow taken as the forward takes it (flow / fh / fw / upsample_mode /
 * flow_mul as there).  grad_cat: [B, cat_channels, H, W]; the ch_* layout must be the forward's.  grad_x: [B, 2C, H, W]
 * and grad_flow: [B, 2, fh, fw] (the gradient of the quarter-resolution flow for upsample_mode 1 / 2), contiguous, fully
 * overwritten.  The composition of the reference modules' own backward passes (torch.cat, the division, ChannelNorm
 * with its 1e-9, the subtraction, Resample2d's K6 scatter and K7 flow gradient, then nn.Upsample's backward times
 * flow_mul) in one kernel plus the transpose of the scatter scratch (grad_x) and, for upsample_mode 1, a pass that adds
 * the per-tile partial sums of the upsample's adjoint (grad_flow).  The full-resolution flow gradient is never written
 * to memory, and grad_flow is bit-identical from run to run (no atomics touch it) and whether or not grad_x is wanted.
 * Either gradient may be NULL: no grad_x = no scatter (and no scratch fill, no transpose), no grad_flow = no K7; both
 * NULL is a successful no-op, as is B = 0.
 * workspace: fn2b200_warp_concat_backward_up_workspace(B, C, H, W, upsample_mode, grad_x != NULL) bytes, 16-byte
 * aligned (0 bytes, and NULL is fine, for upsample_mode 0 / 2 without grad_x).
 */
size_t fn2b200_warp_concat_backward_up_workspace(int B, int C, int H, int W, int upsample_mode, int need_x);
int fn2b200_warp_concat_backward_up(const float *x, const int64_t *xstride, int C, const float *flow, int fh, int fw,
                                    int upsample_mode, float flow_mul, const float *grad_cat, int cat_channels, int ch_x,
                                    int n_x, int ch_warped, int ch_flow, float flow_div, int ch_flow_norm,
                                    int ch_diff_norm, float *grad_x, float *grad_flow, void *workspace,
                                    size_t workspace_bytes, int B, int H, int W, void *stream);

/*
 * fn2b200_warp_concat_backward_up for a full-resolution flow (upsample_mode 0, fh = H, fw = W) with both gradients
 * required (NULL grad_x / grad_flow is an error here).  workspace: fn2b200_warp_concat_backward_workspace(B, C, H, W)
 * = fn2b200_warp_concat_backward_up_workspace(B, C, H, W, 0, 1) bytes, 16-byte aligned.
 */
size_t fn2b200_warp_concat_backward_workspace(int B, int C, int H, int W);
int fn2b200_warp_concat_backward(const float *x, const int64_t *xstride, int C, const float *flow, const float *grad_cat,
                                 int cat_channels, int ch_x, int n_x, int ch_warped, int ch_flow, float flow_div,
                                 int ch_flow_norm, int ch_diff_norm, float *grad_x, float *grad_flow, void *workspace,
                                 size_t workspace_bytes, int B, int H, int W, void *stream);

/* input1: [B,C,H,W]; output: [B,1,H,W] = sqrt(sum_c x^2).  norm_deg is ignored (reference: same). */
int fn2b200_channelnorm_forward(const float *input1, float *output, int B, int C, int H, int W,
                                int norm_deg, void *stream);

/* grad_input1[b,c,p] = grad_output[b,p] * input1[b,c,p] / (output[b,p] + 1e-9). */
int fn2b200_channelnorm_backward(const float *input1, const float *output,
                                 const float *grad_output, float *grad_input1, int B, int C,
                                 int H, int W, int norm_deg, void *stream);

/*
 * 16-bit storage variants of ChannelNorm (dtype: 1 = fp16, 2 = bf16; tensors of that type, fp32
 * arithmetic inside).  The reference dispatches these kernels on half as well
 * (channelnorm_kernel.cu:111,152); ChannelNorm is the one custom layer fed fp16 in --fp16 mode.
 */
int fn2b200_channelnorm_forward_16(const void *input1, void *output, int B, int C, int H, int W, int norm_deg,
                                   int dtype, void *stream);
int fn2b200_channelnorm_backward_16(const void *input1, const void *output, const void *grad_output,
                                    void *grad_input1, int B, int C, int H, int W, int norm_deg, int dtype,
                                    void *stream);

/*
 * Introspection for benchmarks/tests: the kernel family a correlation forward runs for these parameters, given 16-byte
 * aligned pointers and a large-enough workspace (FN2B200_CORR_FWD honoured).  0 = generic gather kernels, 1 = TMA-tiled
 * FP32-FMA kernels, 2 = tensor cores (wgmma).  The backward follows the same rule with FN2B200_CORR_BWD.  A call
 * without the workspace cannot run family 2, one with misaligned pointers not family 1; it then runs the next family
 * whose conditions hold.  -1: invalid parameters.
 */
int fn2b200_correlation_path(int C, int H, int W, int pad_size, int kernel_size,
                             int max_displacement, int stride1, int stride2);

/* Number of kernel launches (ours) issued by this library in this process so far (statistics). */
uint64_t fn2b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FN2B200_H_ */
