// capi.cu -- extern "C" boundary of libfn2b200 (see include/fn2b200.h for the contract).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace fn2 {

// kr, dr, ds, D, oH, oW of a correlation with parameters already checked (s1, s2 >= 1).
static void corr_geometry(CorrParams &p, int C, int H, int W, int pad, int k, int md, int s1, int s2) {
    p.C = C; p.H = H; p.W = W;
    p.pad = pad; p.k = k; p.md = md; p.s1 = s1; p.s2 = s2;
    p.kr = (k - 1) / 2;
    p.dr = md / s2;
    p.ds = 2 * p.dr + 1;
    p.D = p.ds * p.ds;
    int br = p.kr + md;
    // correlation_cuda.cc:33-34 -- float ceil of a float division
    p.oH = (int)ceilf((float)(H + 2 * pad - 2 * br) / (float)s1);
    p.oW = (int)ceilf((float)(W + 2 * pad - 2 * br) / (float)s1);
}

static int fill_corr_params(CorrParams &p, int B, int C, int H, int W, int pad, int k, int md,
                            int s1, int s2) {
    if (B < 0 || C <= 0 || H <= 0 || W <= 0)
        return fail(FN2B200_EINVAL, "correlation: bad input shape [%d,%d,%d,%d]", B, C, H, W);
    if (pad < 0 || k < 1 || md < 0 || s1 < 1 || s2 < 1)
        return fail(FN2B200_EINVAL,
                    "correlation: bad parameters pad=%d kernel_size=%d max_displacement=%d "
                    "stride1=%d stride2=%d", pad, k, md, s1, s2);
    p = CorrParams{};
    p.B = B;
    corr_geometry(p, C, H, W, pad, k, md, s1, s2);
    if (p.oH <= 0 || p.oW <= 0)
        return fail(FN2B200_EINVAL, "correlation: empty output (%d x %d); pad_size too small for "
                    "max_displacement/kernel_size", p.oH, p.oW);
    if ((int64_t)B * C * H * W >= (1LL << 31) || (int64_t)B * p.D * p.oH * p.oW >= (1LL << 31))
        return fail(FN2B200_EINVAL, "correlation: tensor exceeds 2^31 elements");
    return 0;
}

// Every entry point's D correlation planes are channels [ch_offset, ch_offset + D) of a [B, cat_channels, oH, oW] buffer
// (forward output, backward gradOutput) under LeakyReLU(leaky); the plain and *_ws ones use cat_channels = D, 0, 1.
static int place_corr(CorrParams &p, const char *who, int cat_channels, int ch_offset, float leaky) {
    if (ch_offset < 0 || cat_channels < ch_offset + p.D)
        return fail(FN2B200_EINVAL, "%s: channels [%d, %d) do not fit a %d-channel buffer", who, ch_offset,
                    ch_offset + p.D, cat_channels);
    if ((int64_t)p.B * cat_channels * p.oH * p.oW >= (1LL << 31))
        return fail(FN2B200_EINVAL, "%s: tensor exceeds 2^31 elements", who);
    p.out_bstride = p.g_bstride = (long)cat_channels * p.oH * p.oW;
    p.leaky = leaky;
    return 0;
}

// FN2B200_CORR_FWD / FN2B200_CORR_BWD = "fma" keeps that direction on the FP32-FMA kernels; "tc" (default) lets it use
// tensor cores.  Read per call: no cached state.
static bool tc_enabled(bool backward) {
    const char *e = getenv(backward ? "FN2B200_CORR_BWD" : "FN2B200_CORR_FWD");
    return !(e && (e[0] == 'f' || e[0] == 'F'));
}

enum CorrFamily { CORR_GENERIC = 0, CORR_TILED = 1, CORR_TC = 2 };      // the codes of fn2b200_correlation_path

// The one rule that picks a correlation kernel family.  Tensor cores: a supported configuration, the direction's
// environment switch and a large-enough workspace.  TMA-tiled FP32 FMA: a supported configuration and 16-byte aligned
// operands (tensor-map bases and vector stores).  Everything else runs on the generic kernels.
static CorrFamily corr_family(const CorrParams &p, bool backward, bool workspace_ok, bool aligned) {
    if (workspace_ok && tc_enabled(backward) && corr_tc_supported(p)) return CORR_TC;
    if (aligned && corr_tiled_supported(p)) return CORR_TILED;
    return CORR_GENERIC;
}

static bool aligned16(const void *q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

// Every correlation forward; dense = the plain [B, D, oH, oW] output.  `who` (the public name) prefixes error messages.
static int corr_forward(const char *who, const float *in1, const float *in2, float *cat, bool dense, int cat_channels,
                        int ch_offset, float leaky, int B, int C, int H, int W, int pad, int k, int md, int s1, int s2,
                        void *workspace, size_t workspace_bytes, void *stream) {
    CorrParams p;
    int rc = fill_corr_params(p, B, C, H, W, pad, k, md, s1, s2);
    if (rc || (rc = place_corr(p, who, dense ? p.D : cat_channels, ch_offset, leaky))) return rc;
    if (B == 0) return 0;
    if (!in1 || !in2 || !cat) return fail(FN2B200_ENULL, "%s: null pointer", who);
    float *out = cat + (long)ch_offset * p.oH * p.oW;
    if ((rc = bind_device_of(in1))) return rc;
    // the tiled epilogue's 16-byte stores also need the output's batch stride to be a multiple of 4 elements
    const bool aligned = aligned16(in1) && aligned16(in2) && aligned16(out) && !(p.out_bstride & 3);
    cudaStream_t st = (cudaStream_t)stream;
    switch (corr_family(p, false, workspace && workspace_bytes >= corr_tc_workspace_bytes(p), aligned)) {
    case CORR_TC: return corr_forward_tc(in1, in2, out, p, workspace, workspace_bytes, st);
    case CORR_TILED: return corr_forward_tiled(in1, in2, out, p, st);
    default: return corr_forward_generic(in1, in2, out, p, st);
    }
}

// Every correlation backward, as corr_forward; cat (the forward's activated output) is read only when leaky != 1.
static int corr_backward(const char *who, const float *in1, const float *in2, const float *grad_cat, const float *cat,
                         bool dense, int cat_channels, int ch_offset, float leaky, float *gin1, float *gin2, int B, int C,
                         int H, int W, int pad, int k, int md, int s1, int s2, void *workspace, size_t workspace_bytes,
                         int workspace_has_split, void *stream) {
    CorrParams p;
    int rc = fill_corr_params(p, B, C, H, W, pad, k, md, s1, s2);
    if (rc) return rc;
    if (!(leaky >= 0.f))
        return fail(FN2B200_EINVAL, "%s: leaky_slope %g < 0 (the sign of the activated output no longer tells which "
                    "side of 0 the correlation was on)", who, (double)leaky);
    if ((rc = place_corr(p, who, dense ? p.D : cat_channels, ch_offset, leaky))) return rc;
    if (s1 != 1)
        return fail(FN2B200_EUNSUPPORTED, "%s: stride1=%d unsupported (the reference kernels index out of bounds for "
                    "stride1 != 1, correlation_cuda_kernel.cu:163-164 vs :520)", who, s1);
    if (B == 0) return 0;
    const bool act = leaky != 1.f;
    if (!in1 || !in2 || !grad_cat || (act && !cat)) return fail(FN2B200_ENULL, "%s: null pointer", who);
    if (!gin1 && !gin2) return 0;
    const long offset = (long)ch_offset * p.oH * p.oW;
    const float *gout = grad_cat + offset;
    p.act = act ? cat + offset : nullptr;
    if ((rc = bind_device_of(in1))) return rc;
    const bool aligned = aligned16(in1) && aligned16(in2) && aligned16(gout) && (!gin1 || aligned16(gin1)) &&
                         (!gin2 || aligned16(gin2)) && (!p.act || aligned16(p.act));
    cudaStream_t st = (cudaStream_t)stream;
    switch (corr_family(p, true, workspace && workspace_bytes >= corr_tc_workspace_bytes(p), aligned)) {
    case CORR_TC:
        return corr_backward_tc(in1, in2, gout, gin1, gin2, p, workspace, workspace_bytes, workspace_has_split, st);
    case CORR_TILED: return corr_backward_tiled(in1, in2, gout, gin1, gin2, p, st);
    default: return corr_backward_generic(in1, in2, gout, gin1, gin2, p, st);
    }
}

}  // namespace fn2

using namespace fn2;

extern "C" {

int fn2b200_version(void) { return FN2B200_VERSION; }

const char *fn2b200_last_error(void) { return last_error_text(); }
uint64_t fn2b200_launch_count(void) { return launches_so_far(); }

int fn2b200_correlation_out_shape(int C, int H, int W, int pad, int k, int md, int s1, int s2,
                                  int *D, int *oH, int *oW) {
    // unlike fill_corr_params: any B, and empty outputs are reported rather than refused
    if (C <= 0 || H <= 0 || W <= 0 || pad < 0 || k < 1 || md < 0 || s1 < 1 || s2 < 1)
        return fail(FN2B200_EINVAL, "correlation_out_shape: bad parameters");
    CorrParams p;
    corr_geometry(p, C, H, W, pad, k, md, s1, s2);
    if (D) *D = p.D;
    if (oH) *oH = p.oH;
    if (oW) *oW = p.oW;
    return 0;
}

int fn2b200_correlation_path(int C, int H, int W, int pad, int k, int md, int s1, int s2) {
    CorrParams p;
    if (fill_corr_params(p, 1, C, H, W, pad, k, md, s1, s2)) return -1;
    return corr_family(p, false, true, true);
}

int fn2b200_correlation_forward(const float *in1, const float *in2, float *out, int B, int C,
                                int H, int W, int pad, int k, int md, int s1, int s2,
                                int corr_type_multiply, void *stream) {
    return fn2b200_correlation_forward_ws(in1, in2, out, B, C, H, W, pad, k, md, s1, s2, corr_type_multiply, nullptr, 0,
                                          stream);
}

size_t fn2b200_correlation_forward_workspace(int B, int C, int H, int W, int pad, int k, int md, int s1,
                                             int s2) {
    CorrParams p;
    if (fill_corr_params(p, B, C, H, W, pad, k, md, s1, s2)) return 0;
    if (!tc_enabled(false)) return 0;
    return corr_tc_workspace_bytes(p);
}

int fn2b200_correlation_forward_ws(const float *in1, const float *in2, float *out, int B, int C, int H,
                                   int W, int pad, int k, int md, int s1, int s2, int corr_type_multiply,
                                   void *workspace, size_t workspace_bytes, void *stream) {
    (void)corr_type_multiply;  // accepted and ignored: correlation_cuda_kernel.cu:369
    return corr_forward("correlation_forward", in1, in2, out, true, 0, 0, 1.f, B, C, H, W, pad, k, md, s1, s2, workspace,
                        workspace_bytes, stream);
}

int fn2b200_correlation_forward_cat(const float *in1, const float *in2, float *cat, int cat_channels, int ch_offset,
                                    float leaky_slope, int B, int C, int H, int W, int pad, int k, int md, int s1, int s2,
                                    int corr_type_multiply, void *workspace, size_t workspace_bytes, void *stream) {
    (void)corr_type_multiply;
    return corr_forward("correlation_forward_cat", in1, in2, cat, false, cat_channels, ch_offset, leaky_slope, B, C, H, W,
                        pad, k, md, s1, s2, workspace, workspace_bytes, stream);
}

int fn2b200_correlation_backward(const float *in1, const float *in2, const float *gout,
                                 float *gin1, float *gin2, int B, int C, int H, int W, int pad,
                                 int k, int md, int s1, int s2, int corr_type_multiply,
                                 void *stream) {
    return fn2b200_correlation_backward_ws(in1, in2, gout, gin1, gin2, B, C, H, W, pad, k, md, s1, s2, corr_type_multiply,
                                           nullptr, 0, 0, stream);
}

size_t fn2b200_correlation_backward_workspace(int B, int C, int H, int W, int pad, int k, int md, int s1,
                                              int s2) {
    CorrParams p;
    if (fill_corr_params(p, B, C, H, W, pad, k, md, s1, s2)) return 0;
    if (!tc_enabled(true)) return 0;
    return corr_tc_workspace_bytes(p);
}

int fn2b200_correlation_backward_ws(const float *in1, const float *in2, const float *gout, float *gin1,
                                    float *gin2, int B, int C, int H, int W, int pad, int k, int md, int s1,
                                    int s2, int corr_type_multiply, void *workspace, size_t workspace_bytes,
                                    int workspace_has_split, void *stream) {
    (void)corr_type_multiply;
    return corr_backward("correlation_backward", in1, in2, gout, nullptr, true, 0, 0, 1.f, gin1, gin2, B, C, H, W, pad, k,
                         md, s1, s2, workspace, workspace_bytes, workspace_has_split, stream);
}

int fn2b200_correlation_backward_cat(const float *in1, const float *in2, const float *grad_cat, const float *cat,
                                     int cat_channels, int ch_offset, float leaky_slope, float *gin1, float *gin2, int B,
                                     int C, int H, int W, int pad, int k, int md, int s1, int s2, int corr_type_multiply,
                                     void *workspace, size_t workspace_bytes, int workspace_has_split, void *stream) {
    (void)corr_type_multiply;
    return corr_backward("correlation_backward_cat", in1, in2, grad_cat, cat, false, cat_channels, ch_offset, leaky_slope,
                         gin1, gin2, B, C, H, W, pad, k, md, s1, s2, workspace, workspace_bytes, workspace_has_split,
                         stream);
}

// shared argument checks of the fused warp-concat entry points
static int check_warp_layout(const char *who, int C, int cat_channels, int ch_x, int n_x, int ch_warped, int ch_flow,
                             float flow_div, int ch_flow_norm, int ch_diff_norm) {
    struct { int ch, n; const char *what; } slots[5] = {{ch_x, n_x, "x"}, {ch_warped, C, "warped"}, {ch_flow, 2, "flow"},
                                                         {ch_flow_norm, 1, "flow norm"}, {ch_diff_norm, 1, "diff norm"}};
    for (int i = 0; i < 5; ++i) {
        if (slots[i].ch < 0) continue;
        if (slots[i].n < 0 || slots[i].ch + slots[i].n > cat_channels)
            return fail(FN2B200_EINVAL, "%s: %s channels [%d, %d) outside the %d-channel output", who, slots[i].what,
                        slots[i].ch, slots[i].ch + slots[i].n, cat_channels);
        for (int j = 0; j < i; ++j)
            if (slots[j].ch >= 0 && slots[i].ch < slots[j].ch + slots[j].n && slots[j].ch < slots[i].ch + slots[i].n)
                return fail(FN2B200_EINVAL, "%s: %s and %s channel ranges overlap", who, slots[i].what, slots[j].what);
    }
    if (ch_x >= 0 && n_x > 2 * C) return fail(FN2B200_EINVAL, "%s: n_x=%d > 2C", who, n_x);
    if (ch_flow >= 0 && flow_div == 0.f) return fail(FN2B200_EINVAL, "%s: flow_div = 0", who);
    return 0;
}

static int check_resample(const char *who, const int64_t *istride, int B, int C, int iH, int iW,
                          int H, int W, int kernel_size) {
    if (B < 0 || C <= 0 || iH <= 0 || iW <= 0 || H <= 0 || W <= 0)
        return fail(FN2B200_EINVAL, "%s: bad shape B=%d C=%d iH=%d iW=%d H=%d W=%d", who, B, C, iH,
                    iW, H, W);
    if (!istride) return fail(FN2B200_ENULL, "%s: null input1 stride array", who);
    if (kernel_size != 1)
        return fail(FN2B200_EUNSUPPORTED,
                    "%s: kernel_size=%d unsupported (the reference's kernel_size > 1 taps are "
                    "unclamped and read out of bounds, resample2d_kernel.cu:54-61)", who, kernel_size);
    if (iH < H || iW < W)
        return fail(FN2B200_EUNSUPPORTED,
                    "%s: input1 spatial dims (%d,%d) smaller than the flow's (%d,%d): the reference "
                    "clamps with the flow dims and would read out of bounds", who, iH, iW, H, W);
    if ((int64_t)B * C * H * W >= (1LL << 31) || (int64_t)B * C * iH * iW >= (1LL << 31))
        return fail(FN2B200_EINVAL, "%s: tensor exceeds 2^31 elements", who);
    return 0;
}

int fn2b200_resample2d_forward(const float *img, const int64_t *istride, const float *flow,
                               float *out, int B, int C, int iH, int iW, int H, int W,
                               int kernel_size, int bilinear, void *stream) {
    int rc = check_resample("resample2d_forward", istride, B, C, iH, iW, H, W, kernel_size);
    if (rc) return rc;
    if (B == 0) return 0;
    if (!img || !flow || !out) return fail(FN2B200_ENULL, "resample2d_forward: null pointer");
    if ((rc = bind_device_of(flow))) return rc;
    FlowSrc fs = {flow, H, W, 0, 1.f};
    WarpOut o = {out, C, -1, 0, 0, -1, -1, -1, 1.f};
    return resample2d_forward_tile(img, istride, nullptr, nullptr, fs, o, B, C, H, W, bilinear, (cudaStream_t)stream);
}

static int check_flow_src(const char *who, const float *flow, int fh, int fw, int mode, int H, int W) {
    if (!flow) return fail(FN2B200_ENULL, "%s: null flow pointer", who);
    if (mode < 0 || mode > 2) return fail(FN2B200_EINVAL, "%s: upsample_mode %d (0 none, 1 bilinear x4, 2 nearest x4)", who, mode);
    if (mode == 0 ? (fh != H || fw != W) : (fh * 4 != H || fw * 4 != W))
        return fail(FN2B200_EINVAL, "%s: flow %d x %d does not match the %d x %d output for upsample_mode %d", who, fh, fw, H, W, mode);
    return 0;
}

int fn2b200_resample2d_forward_up(const float *img, const int64_t *istride, const float *flow, int fh, int fw,
                                  int upsample_mode, float flow_mul, float *out, int B, int C, int H, int W,
                                  void *stream) {
    int rc = check_resample("resample2d_forward_up", istride, B, C, H, W, H, W, 1);
    if (rc) return rc;
    if ((rc = check_flow_src("resample2d_forward_up", flow, fh, fw, upsample_mode, H, W))) return rc;
    if (B == 0) return 0;
    if (!img || !out) return fail(FN2B200_ENULL, "resample2d_forward_up: null pointer");
    if ((rc = bind_device_of(flow))) return rc;
    FlowSrc fs = {flow, fh, fw, upsample_mode, upsample_mode ? flow_mul : 1.f};
    WarpOut o = {out, C, -1, 0, 0, -1, -1, -1, 1.f};
    return resample2d_forward_tile(img, istride, nullptr, nullptr, fs, o, B, C, H, W, 1, (cudaStream_t)stream);
}

int fn2b200_warp_concat_forward(const float *x, const int64_t *xstride, int C, const float *flow, int fh, int fw,
                                int upsample_mode, float flow_mul, float *cat, int cat_channels, int ch_x, int n_x,
                                int ch_warped, int ch_flow, float flow_div, int ch_flow_norm, int ch_diff_norm, int B,
                                int H, int W, void *stream) {
    if (B < 0 || C < 1 || H <= 0 || W <= 0 || cat_channels < 1)
        return fail(FN2B200_EINVAL, "warp_concat_forward: bad shape B=%d C=%d H=%d W=%d cat_channels=%d", B, C, H, W, cat_channels);
    if (!xstride) return fail(FN2B200_ENULL, "warp_concat_forward: null stride array");
    int rc = check_flow_src("warp_concat_forward", flow, fh, fw, upsample_mode, H, W);
    if (rc) return rc;
    if ((rc = check_warp_layout("warp_concat_forward", C, cat_channels, ch_x, n_x, ch_warped, ch_flow, flow_div, ch_flow_norm,
                                ch_diff_norm))) return rc;
    if ((int64_t)B * cat_channels * H * W >= (1LL << 31)) return fail(FN2B200_EINVAL, "warp_concat_forward: tensor exceeds 2^31 elements");
    if (B == 0) return 0;
    if (!x || !cat) return fail(FN2B200_ENULL, "warp_concat_forward: null pointer");
    const float *img1 = x + (int64_t)C * xstride[1];          // x = [img0 | img1] along channels (models.py:124-126)
    if ((rc = bind_device_of(flow))) return rc;
    FlowSrc fs = {flow, fh, fw, upsample_mode, upsample_mode ? flow_mul : 1.f};
    WarpOut o = {cat, cat_channels, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm, flow_div};
    return resample2d_forward_tile(img1, xstride, x, xstride, fs, o, B, C, H, W, 1, (cudaStream_t)stream);
}

int fn2b200_resample2d_backward_ws(const float *img, const int64_t *istride, const float *flow,
                                   const float *gout, float *gimg, float *gflow, int B, int C, int iH, int iW, int H,
                                   int W, int kernel_size, int bilinear, int zero_grad_input1, void *workspace,
                                   size_t workspace_bytes, void *stream);

int fn2b200_resample2d_backward(const float *img, const int64_t *istride, const float *flow,
                                const float *gout, float *gimg, float *gflow, int B, int C,
                                int iH, int iW, int H, int W, int kernel_size, int bilinear,
                                int zero_grad_input1, void *stream) {
    return fn2b200_resample2d_backward_ws(img, istride, flow, gout, gimg, gflow, B, C, iH, iW, H, W, kernel_size, bilinear,
                                          zero_grad_input1, nullptr, 0, stream);
}

size_t fn2b200_warp_concat_backward_workspace(int B, int C, int H, int W) {
    return fn2b200_warp_concat_backward_up_workspace(B, C, H, W, 0, 1);
}

size_t fn2b200_warp_concat_backward_up_workspace(int B, int C, int H, int W, int upsample_mode, int need_x) {
    if (B <= 0 || C < 1 || C > 3 || H <= 0 || W <= 0 || upsample_mode < 0 || upsample_mode > 2) return 0;
    return warp_concat_backward_workspace_bytes(B, H, W, upsample_mode, need_x != 0);
}

// The two backward entry points: `plain` is fn2b200_warp_concat_backward (full-resolution flow, both gradients
// required, its own message prefix and workspace query); otherwise fn2b200_warp_concat_backward_up.
static int warp_concat_backward(bool plain, const float *x, const int64_t *xstride, int C, const float *flow, int fh,
                                int fw, int upsample_mode, float flow_mul, const float *grad_cat, int cat_channels,
                                int ch_x, int n_x, int ch_warped, int ch_flow, float flow_div, int ch_flow_norm,
                                int ch_diff_norm, float *grad_x, float *grad_flow, void *workspace, size_t workspace_bytes,
                                int B, int H, int W, void *stream) {
    const char *who = plain ? "warp_concat_backward" : "warp_concat_backward_up";
    if (B < 0 || C < 1 || H <= 0 || W <= 0 || cat_channels < 1)
        return fail(FN2B200_EINVAL, "%s: bad shape B=%d C=%d H=%d W=%d cat_channels=%d", who, B, C, H, W, cat_channels);
    if (C > 3) return fail(FN2B200_EUNSUPPORTED, "%s: C=%d > 3 (the interleaved gradient scratch holds 4 floats per pixel)", who, C);
    if (!xstride) return fail(FN2B200_ENULL, "%s: null stride array", who);
    int rc = plain ? 0 : check_flow_src(who, flow, fh, fw, upsample_mode, H, W);
    if (rc) return rc;
    if ((rc = check_warp_layout(who, C, cat_channels, ch_x, n_x, ch_warped, ch_flow, flow_div, ch_flow_norm, ch_diff_norm)))
        return rc;
    if ((int64_t)B * cat_channels * H * W >= (1LL << 31)) return fail(FN2B200_EINVAL, "%s: tensor exceeds 2^31 elements", who);
    if (B == 0) return 0;
    if (plain ? (!x || !flow || !grad_cat || !grad_x || !grad_flow) : (grad_x || grad_flow) && (!x || !grad_cat))
        return fail(FN2B200_ENULL, "%s: null pointer", who);
    if (!grad_x && !grad_flow) return 0;          // no gradient wanted
    const size_t need = warp_concat_backward_workspace_bytes(B, H, W, upsample_mode, grad_x != nullptr);
    if ((need && !workspace) || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 15))
        return fail(FN2B200_EINVAL, "%s: needs a 16-byte aligned workspace of fn2b200_%s_workspace() bytes", who, who);
    if ((rc = bind_device_of(flow))) return rc;
    const FlowSrc fs = {flow, fh, fw, upsample_mode, upsample_mode ? flow_mul : 1.f};
    WarpOut o = {nullptr, cat_channels, ch_x, n_x, ch_warped, ch_flow, ch_flow_norm, ch_diff_norm, flow_div};
    return warp_concat_backward_tile(x, xstride, fs, grad_cat, o, grad_x, grad_flow, workspace, B, C, H, W,
                                     (cudaStream_t)stream);
}

int fn2b200_warp_concat_backward(const float *x, const int64_t *xstride, int C, const float *flow, const float *grad_cat,
                                 int cat_channels, int ch_x, int n_x, int ch_warped, int ch_flow, float flow_div,
                                 int ch_flow_norm, int ch_diff_norm, float *grad_x, float *grad_flow, void *workspace,
                                 size_t workspace_bytes, int B, int H, int W, void *stream) {
    return warp_concat_backward(true, x, xstride, C, flow, H, W, 0, 1.f, grad_cat, cat_channels, ch_x, n_x, ch_warped,
                                ch_flow, flow_div, ch_flow_norm, ch_diff_norm, grad_x, grad_flow, workspace,
                                workspace_bytes, B, H, W, stream);
}

int fn2b200_warp_concat_backward_up(const float *x, const int64_t *xstride, int C, const float *flow, int fh, int fw,
                                    int upsample_mode, float flow_mul, const float *grad_cat, int cat_channels, int ch_x,
                                    int n_x, int ch_warped, int ch_flow, float flow_div, int ch_flow_norm,
                                    int ch_diff_norm, float *grad_x, float *grad_flow, void *workspace,
                                    size_t workspace_bytes, int B, int H, int W, void *stream) {
    return warp_concat_backward(false, x, xstride, C, flow, fh, fw, upsample_mode, flow_mul, grad_cat, cat_channels, ch_x,
                                n_x, ch_warped, ch_flow, flow_div, ch_flow_norm, ch_diff_norm, grad_x, grad_flow,
                                workspace, workspace_bytes, B, H, W, stream);
}

size_t fn2b200_resample2d_backward_workspace(const int64_t *istride, int B, int C, int iH, int iW, int H, int W) {
    if (!istride || B <= 0 || C <= 0 || C > 3 || H <= 0 || W <= 0) return 0;
    return resample2d_backward_workspace_bytes(B, iH, iW);
}

int fn2b200_resample2d_backward_ws(const float *img, const int64_t *istride, const float *flow,
                                   const float *gout, float *gimg, float *gflow, int B, int C, int iH, int iW, int H,
                                   int W, int kernel_size, int bilinear, int zero_grad_input1, void *workspace,
                                   size_t workspace_bytes, void *stream) {
    (void)bilinear;  // the reference's backward ignores it (resample2d_kernel.cu:75-198)
    int rc = check_resample("resample2d_backward", istride, B, C, iH, iW, H, W, kernel_size);
    if (rc) return rc;
    if (B == 0) return 0;
    if (!img || !flow || !gout) return fail(FN2B200_ENULL, "resample2d_backward: null pointer");
    if (!gimg && !gflow) return 0;
    if ((rc = bind_device_of(flow))) return rc;
    // zero_grad_input1 == 0: the caller zero-filled grad_input1 and expects accumulation into it (resample2d.py:31)
    return resample2d_backward_tile(img, istride, flow, gout, gimg, gflow, workspace, workspace_bytes, zero_grad_input1, B,
                                    C, iH, iW, H, W, (cudaStream_t)stream);
}

int fn2b200_channelnorm_forward(const float *in, float *out, int B, int C, int H, int W,
                                int norm_deg, void *stream) {
    (void)norm_deg;  // ignored by the reference kernels too (channelnorm_kernel.cu:18-60)
    if (B < 0 || C <= 0 || H <= 0 || W <= 0)
        return fail(FN2B200_EINVAL, "channelnorm_forward: bad shape [%d,%d,%d,%d]", B, C, H, W);
    if ((int64_t)B * C * H * W >= (1LL << 31))
        return fail(FN2B200_EINVAL, "channelnorm_forward: tensor exceeds 2^31 elements");
    if (B == 0) return 0;
    if (!in || !out) return fail(FN2B200_ENULL, "channelnorm_forward: null pointer");
    if (int rc = bind_device_of(in)) return rc;
    return channelnorm_forward(in, out, B, C, H, W, (cudaStream_t)stream);
}

int fn2b200_channelnorm_backward(const float *in, const float *out, const float *gout, float *gin,
                                 int B, int C, int H, int W, int norm_deg, void *stream) {
    (void)norm_deg;
    if (B < 0 || C <= 0 || H <= 0 || W <= 0)
        return fail(FN2B200_EINVAL, "channelnorm_backward: bad shape [%d,%d,%d,%d]", B, C, H, W);
    if ((int64_t)B * C * H * W >= (1LL << 31))
        return fail(FN2B200_EINVAL, "channelnorm_backward: tensor exceeds 2^31 elements");
    if (B == 0) return 0;
    if (!in || !out || !gout || !gin)
        return fail(FN2B200_ENULL, "channelnorm_backward: null pointer");
    if (int rc = bind_device_of(in)) return rc;
    return channelnorm_backward(in, out, gout, gin, B, C, H, W, (cudaStream_t)stream);
}

int fn2b200_channelnorm_forward_16(const void *in, void *out, int B, int C, int H, int W, int norm_deg,
                                   int dtype, void *stream) {
    (void)norm_deg;
    if (B < 0 || C <= 0 || H <= 0 || W <= 0 || (dtype != 1 && dtype != 2))
        return fail(FN2B200_EINVAL, "channelnorm_forward_16: bad shape [%d,%d,%d,%d] or dtype %d", B, C, H, W, dtype);
    if ((int64_t)B * C * H * W >= (1LL << 31)) return fail(FN2B200_EINVAL, "channelnorm_forward_16: tensor too large");
    if (B == 0) return 0;
    if (!in || !out) return fail(FN2B200_ENULL, "channelnorm_forward_16: null pointer");
    if (int rc = bind_device_of(in)) return rc;
    return channelnorm_forward_half(in, out, B, C, H, W, dtype, (cudaStream_t)stream);
}

int fn2b200_channelnorm_backward_16(const void *in, const void *out, const void *gout, void *gin, int B, int C,
                                    int H, int W, int norm_deg, int dtype, void *stream) {
    (void)norm_deg;
    if (B < 0 || C <= 0 || H <= 0 || W <= 0 || (dtype != 1 && dtype != 2))
        return fail(FN2B200_EINVAL, "channelnorm_backward_16: bad shape [%d,%d,%d,%d] or dtype %d", B, C, H, W, dtype);
    if ((int64_t)B * C * H * W >= (1LL << 31)) return fail(FN2B200_EINVAL, "channelnorm_backward_16: tensor too large");
    if (B == 0) return 0;
    if (!in || !out || !gout || !gin) return fail(FN2B200_ENULL, "channelnorm_backward_16: null pointer");
    if (int rc = bind_device_of(in)) return rc;
    return channelnorm_backward_half(in, out, gout, gin, B, C, H, W, dtype, (cudaStream_t)stream);
}

}  // extern "C"
