// correlation_generic.cu -- correlation forward/backward for ARBITRARY layer parameters.
//
// Correct-for-everything gather kernels used when the TMA-tiled kernels (correlation_tiled.cu) do
// not cover the configuration (kernel_size > 1, stride1 > 1, unusual displacement grids, widths
// that are not a multiple of 4).  FlowNet2's only configuration (pad=20,k=1,md=20,s1=1,s2=2) never
// takes this path.  Semantics follow the reference formulas
// (correlation_cuda_kernel.cu:73-147, :150-241, :243-334) evaluated directly on the NCHW inputs
// with explicit zero padding -- no padded NHWC scratch tensors, no memsets, one launch per batch.
#include "common.cuh"

namespace fn2 {

// out[n,tc,oy,ox]; one thread per output element, ox fastest (coalesced along x for both inputs).
__global__ void __launch_bounds__(256)
corr_fwd_generic_kernel(const float *__restrict__ in1, const float *__restrict__ in2,
                        float *__restrict__ out, CorrParams p, long total) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    int ox = (int)(idx % p.oW);
    long t = idx / p.oW;
    int oy = (int)(t % p.oH);
    t /= p.oH;
    int tc = (int)(t % p.D);
    int n = (int)(t / p.D);
    int tj = tc / p.ds - p.dr, ti = tc % p.ds - p.dr;
    // unpadded coordinates of the patch centres
    int y1 = oy * p.s1 + p.md - p.pad, x1 = ox * p.s1 + p.md - p.pad;
    int y2 = y1 + tj * p.s2, x2 = x1 + ti * p.s2;
    const long hw = (long)p.H * p.W;
    const float *a = in1 + (long)n * p.C * hw;
    const float *b = in2 + (long)n * p.C * hw;
    float acc = 0.f;
    for (int j = -p.kr; j <= p.kr; ++j) {
        int ya = y1 + j, yb = y2 + j;
        if (ya < 0 || ya >= p.H || yb < 0 || yb >= p.H) continue;
        for (int i = -p.kr; i <= p.kr; ++i) {
            int xa = x1 + i, xb = x2 + i;
            if (xa < 0 || xa >= p.W || xb < 0 || xb >= p.W) continue;
            const float *pa = a + (long)ya * p.W + xa;
            const float *pb = b + (long)yb * p.W + xb;
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
            int c = 0;
            for (; c + 4 <= p.C; c += 4) {
                s0 += __ldg(pa + (c + 0) * hw) * __ldg(pb + (c + 0) * hw);
                s1 += __ldg(pa + (c + 1) * hw) * __ldg(pb + (c + 1) * hw);
                s2 += __ldg(pa + (c + 2) * hw) * __ldg(pb + (c + 2) * hw);
                s3 += __ldg(pa + (c + 3) * hw) * __ldg(pb + (c + 3) * hw);
            }
            for (; c < p.C; ++c) s0 += __ldg(pa + c * hw) * __ldg(pb + c * hw);
            acc += (s0 + s1) + (s2 + s3);
        }
    }
    float v = acc / (float)(p.k * p.k * p.C);
    if (p.leaky != 1.f) v = v > 0.f ? v : v * p.leaky;
    out[(long)n * p.out_bstride + ((long)tc * p.oH + oy) * p.oW + ox] = v;
}

// WHICH == 1: gradInput1 (other = input2); WHICH == 2: gradInput2 (other = input1).  stride1 == 1.
template <int WHICH>
__global__ void __launch_bounds__(256)
corr_bwd_generic_kernel(const float *__restrict__ other, const float *__restrict__ gout,
                        float *__restrict__ gin, CorrParams p, long total) {
    long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    int bx = (int)(idx % p.W);
    long t = idx / p.W;
    int by = (int)(t % p.H);
    t /= p.H;
    int c = (int)(t % p.C);
    int n = (int)(t / p.C);
    // padded coordinates, as in the reference (:163-164)
    int y = by + p.pad, x = bx + p.pad;
    const long hw = (long)p.H * p.W, ohw = (long)p.oH * p.oW;
    const float *src = other + ((long)n * p.C + c) * hw;
    const float *g = gout + (long)n * p.g_bstride;
    const float *ga = p.act ? p.act + (long)n * p.g_bstride : nullptr;
    float acc = 0.f;
    for (int tc = 0; tc < p.D; ++tc) {
        int i2 = (tc % p.ds - p.dr) * p.s2, j2 = (tc / p.ds - p.dr) * p.s2;
        int xmin, xmax, ymin, ymax, yy, xx;
        if (WHICH == 1) {
            xmin = x - p.kr - p.md; xmax = x + p.kr - p.md;
            ymin = y - p.kr - p.md; ymax = y + p.kr - p.md;
            yy = y + j2 - p.pad; xx = x + i2 - p.pad;  // unpadded position in input2
        } else {
            xmin = x - p.kr - p.md - i2; xmax = x + p.kr - p.md - i2;
            ymin = y - p.kr - p.md - j2; ymax = y + p.kr - p.md - j2;
            yy = y - j2 - p.pad; xx = x - i2 - p.pad;  // unpadded position in input1
        }
        if (xmax < 0 || ymax < 0 || xmin >= p.oW || ymin >= p.oH) continue;
        if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;  // zero padding
        xmin = max(0, xmin); xmax = min(p.oW - 1, xmax);
        ymin = max(0, ymin); ymax = min(p.oH - 1, ymax);
        float v = __ldg(src + (long)yy * p.W + xx);
        float w = 0.f;
        const float *gp = g + (long)tc * ohw;
        for (int j = ymin; j <= ymax; ++j)
            for (int i = xmin; i <= xmax; ++i) {
                const long o = (long)j * p.oW + i;
                float gv = __ldg(gp + o);
                // LeakyReLU's derivative per element, before the window sum (bit-identical to masking in torch first)
                if (ga) gv = __ldg(ga + (long)tc * ohw + o) > 0.f ? gv : gv * p.leaky;
                w += gv;
            }
        acc += w * v;
    }
    gin[idx] = acc / (float)(p.k * p.k * p.C);
}

int corr_forward_generic(const float *in1, const float *in2, float *out, const CorrParams &p,
                         cudaStream_t st) {
    long total = (long)p.B * p.D * p.oH * p.oW;
    const int T = 256;
    corr_fwd_generic_kernel<<<(unsigned)((total + T - 1) / T), T, 0, st>>>(in1, in2, out, p, total);
    count_launch();
    return check_launch("correlation_forward(generic)");
}

int corr_backward_generic(const float *in1, const float *in2, const float *gout, float *gin1,
                          float *gin2, const CorrParams &p, cudaStream_t st) {
    long total = (long)p.B * p.C * p.H * p.W;
    const int T = 256;
    unsigned grid = (unsigned)((total + T - 1) / T);
    if (gin1) {
        corr_bwd_generic_kernel<1><<<grid, T, 0, st>>>(in2, gout, gin1, p, total);
        count_launch();
    }
    if (gin2) {
        corr_bwd_generic_kernel<2><<<grid, T, 0, st>>>(in1, gout, gin2, p, total);
        count_launch();
    }
    return check_launch("correlation_backward(generic)");
}

}  // namespace fn2
