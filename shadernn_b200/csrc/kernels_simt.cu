// CUDA-core (SIMT) kernels for sm_90a: the HBM-bound operators (depthwise, pooling, add, norms, layout ops)
// and the generic direct/implicit-GEMM fp32 convolution used where the tcgen05 path does not apply
// (IC = 3 stems, 1-channel ESPCN layers, reflect/replicate padding).
//
// All activation tensors are split-fp16 NHWC (see snnb_internal.h): every kernel reads hi+lo, computes in fp32
// and writes hi/lo. Channel groups of 8 (= one 16-byte vector per plane) are the unit of work; channels in
// [C, Cp) are written as zero so they never pollute a consumer.
//
// Semantics follow the reference's Vulkan compute shaders (cited per kernel; paths relative to the reference repo
// core/data/assets/shaders/).
#include <algorithm>
#include <cstdlib>

#include "snnb_internal.h"

namespace snnb {

// ------------------------------------------------------------------------------------------------------------
// split-fp16 helpers (snnb_internal.h): a 32-bit word holds two consecutive channels of one plane
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 h2_to_f2(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }
// (a, b) -> packed fp16 pair, round to nearest, saturated to +-65504 (one F2FP.SATFINITE.F16.F32.PACK_AB)
__device__ __forceinline__ uint32_t f2_to_h2(float a, float b) {
    uint32_t h;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
    return h;
}

// 8 channels: v[i] = hi[i] + lo[i]
__device__ __forceinline__ void unpack8(const uint4& h, const uint4& l, float v[8]) {
    const uint32_t hh[4] = {h.x, h.y, h.z, h.w}, ll[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float2 a = h2_to_f2(hh[j]), b = h2_to_f2(ll[j]);
        v[2 * j] = a.x + b.x, v[2 * j + 1] = a.y + b.y;
    }
}
// lo == nullptr: the tensor lives in the half-precision storage mode (SNNB_PRECISION_FP16, one plane). The test is uniform
// over the grid.
__device__ __forceinline__ void load8(const __half* __restrict__ hi, const __half* __restrict__ lo, size_t off, float v[8]) {
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi + off));
    const uint4 l = lo ? __ldg(reinterpret_cast<const uint4*>(lo + off)) : make_uint4(0u, 0u, 0u, 0u);
    unpack8(h, l, v);
}

__device__ __forceinline__ void split2(float a, float b, uint32_t& h, uint32_t& l) {
    h               = f2_to_h2(a, b);
    const float2 hf = h2_to_f2(h);
    l               = f2_to_h2(a - hf.x, b - hf.y);
}

__device__ __forceinline__ void store8(__half* __restrict__ hi, __half* __restrict__ lo, size_t off, const float v[8]) {
    uint4 h, l;
    split2(v[0], v[1], h.x, l.x);
    split2(v[2], v[3], h.y, l.y);
    split2(v[4], v[5], h.z, l.z);
    split2(v[6], v[7], h.w, l.w);
    *reinterpret_cast<uint4*>(hi + off) = h;
    if (lo) *reinterpret_cast<uint4*>(lo + off) = l;
}

struct FeedV { // the compact 4-channel copy of a model input (snnb_tensor::feed_hi), or hi == nullptr
    __half* hi;
    __half* lo;
    int H, W, py, px;
    int only; // snnb_tensor::feed_only: the regular planes are neither written nor read
};
// channels 0..3 of image pixel `pix` back from the stem feed
__device__ __forceinline__ void load_feed(const FeedV& f, size_t pix, int H, int W, float v[8]) {
    const int x = (int) (pix % W), y = (int) ((pix / W) % H);
    const size_t n = pix / ((size_t) W * H);
    const size_t off = ((n * f.H + y + f.py) * f.W + x + f.px) * 4;
    const uint2 h = *reinterpret_cast<const uint2*>(f.hi + off);
    const uint2 l = f.lo ? *reinterpret_cast<const uint2*>(f.lo + off) : make_uint2(0u, 0u);
    const float2 h0 = h2_to_f2(h.x), h1 = h2_to_f2(h.y), l0 = h2_to_f2(l.x), l1 = h2_to_f2(l.y);
    v[0] = h0.x + l0.x, v[1] = h0.y + l0.y, v[2] = h1.x + l1.x, v[3] = h1.y + l1.y;
    v[4] = v[5] = v[6] = v[7] = 0.0f;
}
// channels 0..3 of image pixel `pix` (linear n, y, x index of a tensor H x W) into the stem feed (C <= 4: one thread per pixel)
__device__ __forceinline__ void store_feed(const FeedV& f, size_t pix, int H, int W, const float v[8]) {
    const int x = (int) (pix % W), y = (int) ((pix / W) % H);
    const size_t n = pix / ((size_t) W * H);
    const size_t off = ((n * f.H + y + f.py) * f.W + x + f.px) * 4;
    uint2 h, l;
    split2(v[0], v[1], h.x, l.x);
    split2(v[2], v[3], h.y, l.y);
    *reinterpret_cast<uint2*>(f.hi + off) = h;
    if (f.lo) *reinterpret_cast<uint2*>(f.lo + off) = l;
}

__device__ __forceinline__ float load1(const __half* __restrict__ hi, const __half* __restrict__ lo, size_t off) {
    return __half2float(hi[off]) + (lo ? __half2float(lo[off]) : 0.0f);
}
__device__ __forceinline__ void store1(__half* __restrict__ hi, __half* __restrict__ lo, size_t off, float v) {
    uint32_t h, l;
    split2(v, 0.0f, h, l);
    hi[off] = __ushort_as_half((unsigned short) (h & 0xffffu));
    if (lo) lo[off] = __ushort_as_half((unsigned short) (l & 0xffffu));
}

// Activations: ids of conv2dVulkan.cpp:57-71; math of shadertemplate_vk_conv2d.comp:290-340 (SiLU computed
// correctly per element — the reference's 4-pixel kernel reuses pixel 1's sigmoid, SURVEY Q10).
__device__ __noinline__ float slow_act(float v, int act) {
    switch (act) {
    case SNNB_ACT_TANH: return tanhf(v);
    case SNNB_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    case SNNB_ACT_SILU: return v * 1.0f / (1.0f + expf(-v));
    default: return v;
    }
}
// none / relu / relu6 / leakyRelu are one branch-free max/min pair (slope and clip are loop-invariant); the
// transcendental ones go out of line. max(v, v*alpha) is the reference's own leakyRelu form (vk_conv2d.comp:325-330).
__device__ __forceinline__ float apply_act(float v, int act, float alpha) {
    if (act == SNNB_ACT_TANH || act == SNNB_ACT_SIGMOID || act == SNNB_ACT_SILU) return slow_act(v, act);
    const float slope = (act == SNNB_ACT_RELU || act == SNNB_ACT_RELU6) ? 0.0f : (act == SNNB_ACT_LEAKY_RELU ? alpha : 1.0f);
    const float hi    = act == SNNB_ACT_RELU6 ? 6.0f : __int_as_float(0x7f800000);
    return fminf(fmaxf(v, v * slope), hi);
}

// Source coordinate under a padding mode (vk_conv2d.comp:168-218): returns -1 for "reads zero".
__device__ __forceinline__ int src_coord(int s, int n, int mode) {
    if (mode == SNNB_PAD_REPLICATE) return min(max(s, 0), n - 1);
    if (mode == SNNB_PAD_REFLECT) { // one reflection, as the shader does; still outside -> reads zero (never faults)
        s = (s < 0) ? -s : s;
        s = (s >= n) ? 2 * n - 2 - s : s;
    }
    return (s >= 0 && s < n) ? s : -1;
}

struct TV { // kernel-side tensor view
    __half* hi;
    __half* lo;
    int N, H, W, C, Cp;
};
static TV view(const snnb_tensor* t) { return TV {t->hi, t->lo, t->n, t->h, t->w, t->c, t->cp}; }
static FeedV feed_view(const snnb_tensor* t) { return FeedV {t->feed_hi, t->feed_lo, t->feed_h, t->feed_w, t->feed_py, t->feed_px, t->feed_only ? 1 : 0}; }

// ------------------------------------------------------------------------------------------------------------
// Conv2D, fp32 CUDA-core implicit GEMM (shadertemplate_vk_conv2d.comp:148-347; 1x1: vk_conv2d_1x1.comp:68-211).
//   M = N*OH*OW pixels, Ngemm = OC, K = k*k*IC with k index = (ky*k + kx)*IC + ic.
// Block tile 64 pixels x 64 oc, K chunk 16, 128 threads, 4x8 outputs per thread.
// A is gathered from the split-fp16 input (vector path when IC % 8 == 0, scalar otherwise), B is the packed
// fp32 weight matrix [K][OCw] with BN folded. Epilogue: + bias (+ residual) -> activation -> split -> store.
// ------------------------------------------------------------------------------------------------------------
struct ConvKParams {
    TV in, out, res;
    const float* w;
    const float* bias;
    int ocw;
    int k, stride, pad_x, pad_y, pad_mode, act;
    float alpha;
    int OH, OW, K;
    int has_res;
};

constexpr int CV_BM = 64, CV_BN = 64, CV_BK = 16;

__global__ void __launch_bounds__(128) conv2d_simt_kernel(const ConvKParams p) {
    pdl_wait();
    __shared__ __align__(16) float As[CV_BK][CV_BM + 4];
    __shared__ __align__(16) float Bs[CV_BK][CV_BN];

    const int tid = threadIdx.x;
    const int tx = tid & 7, ty = tid >> 3; // 8 x 16
    const long long M   = (long long) p.in.N * p.OH * p.OW;
    const long long m0  = (long long) blockIdx.x * CV_BM;
    const int oc0       = blockIdx.y * CV_BN;
    const int IC        = p.in.C;

    // the pixel this thread gathers A for
    const int a_px  = tid & 63;
    const int a_kh  = tid >> 6; // which half (8 k's) of the 16-wide chunk
    const long long am = m0 + a_px;
    const bool a_valid = am < M;
    int an = 0, aoy = 0, aox = 0;
    if (a_valid) {
        an        = (int) (am / ((long long) p.OH * p.OW));
        int rem   = (int) (am - (long long) an * p.OH * p.OW);
        aoy       = rem / p.OW;
        aox       = rem - aoy * p.OW;
    }
    const int iy0 = aoy * p.stride - p.pad_y, ix0 = aox * p.stride - p.pad_x;
    const bool vec_path = (IC % 8) == 0;

    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

    for (int k0 = 0; k0 < p.K; k0 += CV_BK) {
        // ---- A chunk: As[kk][pixel] ----
        float av[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) av[j] = 0.0f;
        const int kbase = k0 + a_kh * 8;
        if (a_valid && kbase < p.K) {
            if (vec_path) {
                const int tap = kbase / IC, ic = kbase - tap * IC;
                const int ky = tap / p.k, kx = tap - ky * p.k;
                const int sy = src_coord(iy0 + ky, p.in.H, p.pad_mode), sx = src_coord(ix0 + kx, p.in.W, p.pad_mode);
                if (sy >= 0 && sx >= 0) load8(p.in.hi, p.in.lo, (((size_t) an * p.in.H + sy) * p.in.W + sx) * p.in.Cp + ic, av);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int kk = kbase + j;
                    if (kk < p.K) {
                        const int tap = kk / IC, ic = kk - tap * IC;
                        const int ky = tap / p.k, kx = tap - ky * p.k;
                        const int sy = src_coord(iy0 + ky, p.in.H, p.pad_mode), sx = src_coord(ix0 + kx, p.in.W, p.pad_mode);
                        if (sy >= 0 && sx >= 0) av[j] = load1(p.in.hi, p.in.lo, (((size_t) an * p.in.H + sy) * p.in.W + sx) * p.in.Cp + ic);
                    }
                }
            }
        }
        // ---- B chunk: Bs[kk][oc] ----
        float4 bv[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int idx = tid + r * 128;
            const int row = idx >> 4, c4 = idx & 15;
            const int kk = k0 + row;
            bv[r]        = (kk < p.K) ? __ldg(reinterpret_cast<const float4*>(p.w + (size_t) kk * p.ocw + oc0) + c4) : make_float4(0, 0, 0, 0);
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 8; ++j) As[a_kh * 8 + j][a_px] = av[j];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int idx = tid + r * 128;
            *reinterpret_cast<float4*>(&Bs[idx >> 4][(idx & 15) * 4]) = bv[r];
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < CV_BK; ++kk) {
            const float4 a  = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 8]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 8 + 4]);
            const float aa[4] = {a.x, a.y, a.z, a.w};
            const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
        }
    }

    // ---- epilogue ----
    const int oc = oc0 + tx * 8;
    if (oc >= p.out.Cp) return;
    float bias[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bias[j] = p.bias[oc + j];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= M) continue;
        const size_t off = (size_t) m * p.out.Cp + oc;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = acc[i][j] + bias[j];
        if (p.has_res) {
            float r[8];
            load8(p.res.hi, p.res.lo, off, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += r[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (oc + j < p.out.C) ? apply_act(v[j], p.act, p.alpha) : 0.0f;
        store8(p.out.hi, p.out.lo, off, v);
    }
}

int launch_conv2d_simt(snnb_context* ctx, const ConvArgs& a) {
    SNNB_REQUIRE(!a.in->feed_only, "launch_conv2d_simt: the input tensor only exists as a stem feed, which this kernel cannot read");
    ctx->last_kernel = "conv2d_simt_kernel";
    ConvKParams p;
    p.in      = view(a.in);
    p.out     = view(a.out);
    p.has_res = a.residual != nullptr;
    p.res     = a.residual ? view(a.residual) : view(a.out);
    p.w       = a.w->w_f32;
    p.bias    = a.w->bias;
    p.ocw     = a.w->ocw;
    p.k = a.k, p.stride = a.stride, p.pad_x = a.pad_x, p.pad_y = a.pad_y, p.pad_mode = a.pad_mode, p.act = a.act, p.alpha = a.alpha;
    p.OH = a.out->h, p.OW = a.out->w;
    p.K  = a.k * a.k * a.in->c;
    const long long M = (long long) a.out->n * a.out->h * a.out->w;
    dim3 grid((unsigned) ((M + CV_BM - 1) / CV_BM), (unsigned) ((a.out->cp + CV_BN - 1) / CV_BN));
    return launch_done(ctx, launch_k(conv2d_simt_kernel, dim3(grid), dim3(128), 0, ctx->stream, p), "conv2d_simt_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// Depthwise k x k (shadertemplate_vk_depthwise.comp:64-139): window clipped to the input (== zero padding),
// bias, folded BN, activation. One thread = 8 channels x DW_TX consecutive output columns; the k x (stride*(TX-1)+k)
// input patch is streamed through registers row by row so every input vector is loaded once per thread.
// Weights fp32 [k*k][Cp].
// ------------------------------------------------------------------------------------------------------------
struct DwParams {
    TV in, out;
    const float* w;
    const float* bias;
    int k, stride, pad_x, pad_y, act;
    float alpha;
};

template <int K, int S, int TX>
__global__ void __launch_bounds__(128) depthwise_kernel(const DwParams p) {
    pdl_wait();
    const int CG            = p.out.Cp >> 3;
    const int strips        = (p.out.W + TX - 1) / TX;
    const long long total   = (long long) p.out.N * p.out.H * strips * CG;
    const long long gid     = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int cg    = (int) (gid % CG);
    long long r     = gid / CG;
    const int strip = (int) (r % strips);
    r /= strips;
    const int oy = (int) (r % p.out.H);
    const int n  = (int) (r / p.out.H);
    const int c  = cg * 8;
    const int ox0 = strip * TX;

    float wreg[K * K][8];
#pragma unroll
    for (int t = 0; t < K * K; ++t) {
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t) t * p.in.Cp + c));
        const float4 w1 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t) t * p.in.Cp + c) + 1);
        wreg[t][0] = w0.x, wreg[t][1] = w0.y, wreg[t][2] = w0.z, wreg[t][3] = w0.w;
        wreg[t][4] = w1.x, wreg[t][5] = w1.y, wreg[t][6] = w1.z, wreg[t][7] = w1.w;
    }
    float acc[TX][8];
    {
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(p.bias + c));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(p.bias + c) + 1);
#pragma unroll
        for (int t = 0; t < TX; ++t) {
            acc[t][0] = b0.x, acc[t][1] = b0.y, acc[t][2] = b0.z, acc[t][3] = b0.w;
            acc[t][4] = b1.x, acc[t][5] = b1.y, acc[t][6] = b1.z, acc[t][7] = b1.w;
        }
    }
    constexpr int COLS = S * (TX - 1) + K;
    const int ix0 = ox0 * S - p.pad_x, iy0 = oy * S - p.pad_y;
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
        const int iy = iy0 + ky;
        if (iy < 0 || iy >= p.in.H) continue;
        const size_t rowoff = ((size_t) n * p.in.H + iy) * p.in.W;
#pragma unroll
        for (int cx = 0; cx < COLS; ++cx) {
            const int ix = ix0 + cx;
            if (ix < 0 || ix >= p.in.W) continue;
            float v[8];
            load8(p.in.hi, p.in.lo, (rowoff + ix) * p.in.Cp + c, v);
#pragma unroll
            for (int t = 0; t < TX; ++t) {
                const int kx = cx - t * S; // compile-time after unrolling
                if (kx >= 0 && kx < K) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[t][j] = fmaf(wreg[ky * K + kx][j], v[j], acc[t][j]);
                }
            }
        }
    }
#pragma unroll
    for (int t = 0; t < TX; ++t) {
        const int ox = ox0 + t;
        if (ox >= p.out.W) break;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (c + j < p.out.C) ? apply_act(acc[t][j], p.act, p.alpha) : 0.0f;
        store8(p.out.hi, p.out.lo, (((size_t) n * p.out.H + oy) * p.out.W + ox) * p.out.Cp + c, v);
    }
}

// generic (any k / stride): one thread = 8 channels x 1 output pixel
__global__ void __launch_bounds__(128) depthwise_generic_kernel(const DwParams p) {
    pdl_wait();
    const int CG          = p.out.Cp >> 3;
    const long long total = (long long) p.out.N * p.out.H * p.out.W * CG;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int cg = (int) (gid % CG);
    long long r  = gid / CG;
    const int ox = (int) (r % p.out.W);
    r /= p.out.W;
    const int oy = (int) (r % p.out.H);
    const int n  = (int) (r / p.out.H);
    const int c  = cg * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = p.bias[c + j];
    const int ix0 = ox * p.stride - p.pad_x, iy0 = oy * p.stride - p.pad_y;
    for (int ky = 0; ky < p.k; ++ky) {
        const int iy = iy0 + ky;
        if (iy < 0 || iy >= p.in.H) continue;
        for (int kx = 0; kx < p.k; ++kx) {
            const int ix = ix0 + kx;
            if (ix < 0 || ix >= p.in.W) continue;
            float v[8];
            load8(p.in.hi, p.in.lo, (((size_t) n * p.in.H + iy) * p.in.W + ix) * p.in.Cp + c, v);
            const float* wp = p.w + (size_t) (ky * p.k + kx) * p.in.Cp + c;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = fmaf(__ldg(wp + j), v[j], acc[j]);
        }
    }
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (c + j < p.out.C) ? apply_act(acc[j], p.act, p.alpha) : 0.0f;
    store8(p.out.hi, p.out.lo, (((size_t) n * p.out.H + oy) * p.out.W + ox) * p.out.Cp + c, v);
}

int launch_depthwise(snnb_context* ctx, const ConvArgs& a) {
    static const bool no_tma = getenv("SNNB_DW_SIMT") != nullptr; // A/B switch: the CUDA-core kernels below
    if (!no_tma && depthwise_tma_supported(a)) return launch_depthwise_tma(ctx, a);
    ctx->last_kernel = "depthwise_kernel";
    DwParams p;
    p.in = view(a.in), p.out = view(a.out);
    p.w = a.w->w_f32, p.bias = a.w->bias;
    p.k = a.k, p.stride = a.stride, p.pad_x = a.pad_x, p.pad_y = a.pad_y, p.act = a.act, p.alpha = a.alpha;
    const int CG = a.out->cp >> 3;
    if (a.k == 3 && (a.stride == 1 || a.stride == 2)) {
        constexpr int TX      = 4;
        const int strips      = (a.out->w + TX - 1) / TX;
        const long long total = (long long) a.out->n * a.out->h * strips * CG;
        const unsigned blocks = (unsigned) ((total + 127) / 128);
        if (a.stride == 1) return launch_done(ctx, launch_k(depthwise_kernel<3, 1, TX>, dim3(blocks), dim3(128), 0, ctx->stream, p), "depthwise_kernel");
        return launch_done(ctx, launch_k(depthwise_kernel<3, 2, TX>, dim3(blocks), dim3(128), 0, ctx->stream, p), "depthwise_kernel");
    }
    const long long total = (long long) a.out->n * a.out->h * a.out->w * CG;
    return launch_done(ctx, launch_k(depthwise_generic_kernel, dim3((unsigned) ((total + 127) / 128)), dim3(128), 0, ctx->stream, p), "depthwise_generic_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// Max / average pooling (vk_maxpool2d.comp:42-71, vk_avgpool2d.comp:42-69): window origin o*stride (never padded
// top/left, maxpool2dVulkan.cpp:57-60), taps clipped to the input, max starts at -100000, avg divides by the
// number of valid taps. One thread = 8 channels x 1 output pixel.
// ------------------------------------------------------------------------------------------------------------
// K > 0: window size known at compile time, a window row's taps are loaded together (the generic loop keeps only one tap
// in flight per thread and ran at 40% of the HBM roofline on ResNet's 3x3/2 max pool).
template <int K>
__global__ void __launch_bounds__(256) pool_kernel(TV in, TV out, int k, int stride, int avg) {
    pdl_wait();
    if (K > 0) k = K;
    const int CG          = out.Cp >> 3;
    const long long total = (long long) out.N * out.H * out.W * CG;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int cg = (int) (gid % CG);
    long long r  = gid / CG;
    const int ox = (int) (r % out.W);
    r /= out.W;
    const int oy = (int) (r % out.H);
    const int n  = (int) (r / out.H);
    const int c  = cg * 8;
    const int sx = ox * stride, sy = oy * stride;
    const int efx = min(k, in.W - sx), efy = min(k, in.H - sy);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = avg ? 0.0f : -100000.0f;
    float num = 0.0f;
    if (K > 0) {
        // one window row at a time: its K taps' loads are issued before any is consumed (K x 2 x 16 B in flight per thread) and
        // the register footprint stays small enough for 5+ resident blocks per SM; clipped taps re-read the window origin
        constexpr int KW = K > 0 ? K : 1;
#pragma unroll
        for (int fy = 0; fy < KW; ++fy) {
            uint4 th[KW], tl[KW];
            const bool oky = fy < efy;
#pragma unroll
            for (int fx = 0; fx < KW; ++fx) {
                const bool ok  = oky && fx < efx;
                const size_t o = (((size_t) n * in.H + sy + (ok ? fy : 0)) * in.W + sx + (ok ? fx : 0)) * in.Cp + c;
                th[fx] = __ldg(reinterpret_cast<const uint4*>(in.hi + o));
                tl[fx] = in.lo ? __ldg(reinterpret_cast<const uint4*>(in.lo + o)) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int fx = 0; fx < KW; ++fx) {
                if (oky && fx < efx) {
                    float v[8];
                    unpack8(th[fx], tl[fx], v);
                    if (avg) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[j] += v[j];
                        num += 1.0f;
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], v[j]);
                    }
                }
            }
        }
    } else {
        for (int fy = 0; fy < efy; ++fy)
            for (int fx = 0; fx < efx; ++fx) {
                float v[8];
                load8(in.hi, in.lo, (((size_t) n * in.H + sy + fy) * in.W + sx + fx) * in.Cp + c, v);
                if (avg) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] += v[j];
                    num += 1.0f;
                } else {
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j], v[j]);
                }
            }
    }
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (c + j < out.C) ? (avg ? acc[j] / num : acc[j]) : 0.0f;
    store8(out.hi, out.lo, (((size_t) n * out.H + oy) * out.W + ox) * out.Cp + c, v);
}

// Global average pool (AveragePooling2D with pool == H == W, stride 1, valid — how the converter emits GAP,
// tools/convertTool/layers/supportedLayers/averagepooling2d.py:40-55): one warp per (n, 8-channel group).
__global__ void __launch_bounds__(256) global_avgpool_kernel(TV in, TV out) {
    pdl_wait();
    const int CG   = out.Cp >> 3;
    const int warp = (int) (((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (warp >= in.N * CG) return;
    const int n = warp / CG, c = (warp % CG) * 8;
    const int HW = in.H * in.W;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
    // sequential-in-pixel-order partial sums per lane, then a fixed-shape tree: deterministic
    for (int px = lane; px < HW; px += 32) {
        float v[8];
        load8(in.hi, in.lo, ((size_t) n * HW + px) * in.Cp + c, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    if (lane == 0) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (c + j < out.C) ? acc[j] / (float) HW : 0.0f;
        store8(out.hi, out.lo, (size_t) n * out.Cp + c, v);
    }
}

// Classifier head in one launch: global average pool (AveragePooling2D with pool == H == W) -> Dense (+ activation / softmax),
// i.e. the tail of ResNet-18 (7x7x512 -> 10). Four tiny launches (pool, 1x1 tensor-core GEMM for a single tile, softmax) cost
// more in ramp-up than in work. One CTA per image: pooled vector in shared memory (sequential sum per channel, deterministic),
// one warp per output unit (lanes over input channels, shuffle tree), then the activation or a max-subtracted softmax
// (cpulayer.h:175-191). Weights fp32 [IC][OCw] (the CUDA-core conv layout).
// r02: 1024 threads and a Dense phase with lanes over the UNITS (coalesced weight rows, independent loads): the r01 version (256
// threads, one warp per unit striding the channels) was a chain of ~45 dependent L2 round trips = 16 us for 0.3 MFLOP.
constexpr int GD_THREADS = 1024;
__global__ void __launch_bounds__(GD_THREADS) gap_dense_kernel(TV in, TV out, const float* __restrict__ w, int ocw, const float* __restrict__ bias, int act, float alpha,
                                                               int softmax, int parts) {
    pdl_wait();
    extern __shared__ float hs[]; // [parts][in.Cp] partial sums (row 0 becomes the pooled vector), [32 warps][out.Cp] Dense partials, [out.Cp] logits
    const int n = blockIdx.x, HW = in.H * in.W, CG = in.Cp >> 3;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = GD_THREADS / 32;
    float* xs     = hs; // `parts` pixel ranges are summed by different threads
    float* red    = hs + parts * in.Cp;
    float* logits = red + nwarps * out.Cp;
    for (int item = threadIdx.x; item < CG * parts; item += blockDim.x) {
        const int cg = item % CG, part = item / CG;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
        int px = part;
        for (; px + 3 * parts < HW; px += 4 * parts) { // four independent loads in flight; summed in pixel order (deterministic)
            float v[4][8];
#pragma unroll
            for (int u = 0; u < 4; ++u) load8(in.hi, in.lo, ((size_t) n * HW + px + u * parts) * in.Cp + cg * 8, v[u]);
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] += v[u][j];
        }
        for (; px < HW; px += parts) {
            float v[8];
            load8(in.hi, in.lo, ((size_t) n * HW + px) * in.Cp + cg * 8, v);
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] += v[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) xs[part * in.Cp + cg * 8 + j] = acc[j];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < in.Cp; c += blockDim.x) { // fixed order over the parts: deterministic
        float t = xs[c];
        for (int q = 1; q < parts; ++q) t += xs[q * in.Cp + c];
        xs[c] = t / (float) HW;
    }
    __syncthreads();
    // Dense: warp `warp` takes the channels c = warp, warp + 32, ...; its lanes take the units oc = lane, lane + 32, ... (<= 8 per lane:
    // out.C <= 256): every load of a weight row is coalesced and the loads of different channels are independent
    {
        float part[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) part[k] = 0.0f;
        int c = warp;
        for (; c + 3 * nwarps < in.C; c += 4 * nwarps) { // four weight rows in flight per lane (each an L2 round trip), summed in channel order
            float wv[4][8];
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int k = 0; k < 8; ++k) wv[u][k] = (lane + 32 * k < out.C) ? __ldg(w + (size_t) (c + u * nwarps) * ocw + lane + 32 * k) : 0.0f;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float xv = xs[c + u * nwarps];
#pragma unroll
                for (int k = 0; k < 8; ++k) part[k] = fmaf(xv, wv[u][k], part[k]);
            }
        }
        for (; c < in.C; c += nwarps) {
            const float xv    = xs[c];
            const float* wrow = w + (size_t) c * ocw;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int oc = lane + 32 * k;
                if (oc < out.C) part[k] = fmaf(xv, __ldg(wrow + oc), part[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int oc = lane + 32 * k;
            if (oc < out.C) red[warp * out.Cp + oc] = part[k];
        }
    }
    __syncthreads();
    for (int oc = threadIdx.x; oc < out.C; oc += blockDim.x) { // warps added in order: deterministic
        float s = red[oc];
        for (int q = 1; q < nwarps; ++q) s += red[q * out.Cp + oc];
        logits[oc] = softmax ? s + bias[oc] : apply_act(s + bias[oc], act, alpha);
    }
    __syncthreads();
    if (softmax && warp == 0) { // max-subtracted softmax over the units, fixed-shape tree
        float m = -3.402823466e+38f;
        for (int oc = lane; oc < out.C; oc += 32) m = fmaxf(m, logits[oc]);
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float z = 0.0f;
        for (int oc = lane; oc < out.C; oc += 32) z += expf(logits[oc] - m);
        for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
        for (int oc = lane; oc < out.C; oc += 32) logits[oc] = expf(logits[oc] - m) / z;
    }
    __syncthreads();
    for (int oc = threadIdx.x; oc < out.Cp; oc += blockDim.x) store1(out.hi, out.lo, (size_t) n * out.Cp + oc, oc < out.C ? logits[oc] : 0.0f);
}

// pixel ranges per channel group, limited by the 48 KB of shared memory available without opt-in; 0 = does not fit
static int gap_dense_parts(const snnb_tensor* in, const snnb_tensor* out) {
    int parts = std::max(1, std::min(GD_THREADS / (in->cp >> 3), 8));
    while (parts > 1 && (size_t) (parts * in->cp + (GD_THREADS / 32 + 1) * out->cp) * sizeof(float) > 48 * 1024) --parts;
    return (size_t) (parts * in->cp + (GD_THREADS / 32 + 1) * out->cp) * sizeof(float) > 48 * 1024 ? 0 : parts;
}
bool gap_dense_supported(const snnb_tensor* in, const snnb_tensor* out, const snnb_weights* w) {
    return w && w->w_f32 && in->h * in->w >= 4 && in->cp <= 4096 && out->c <= 256 && out->h * out->w == 1 && in->n == out->n && gap_dense_parts(in, out) > 0;
}
int launch_gap_dense(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, const snnb_weights* w, int act, float alpha, bool softmax) {
    ctx->last_kernel = "gap_dense_kernel";
    const int parts   = gap_dense_parts(in, out);
    SNNB_REQUIRE(parts > 0, "launch_gap_dense: the head does not fit in shared memory");
    const size_t smem = (size_t) (parts * in->cp + (GD_THREADS / 32 + 1) * out->cp) * sizeof(float);
    return launch_done(ctx, launch_k(gap_dense_kernel, dim3((unsigned) in->n), dim3(GD_THREADS), smem, ctx->stream, view(in), view(out), (const float*) w->w_f32, w->ocw, (const float*) w->bias, act, alpha,
             softmax ? 1 : 0, parts), "gap_dense_kernel");
}

int launch_pool(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, int k, int stride, bool avg) {
    ctx->last_kernel = "pool_kernel";
    TV vi = view(in), vo = view(out);
    if (avg && out->h == 1 && out->w == 1 && k >= in->h && k >= in->w && in->h * in->w >= 16) {
        const long long warps = (long long) in->n * (out->cp >> 3);
        return launch_done(ctx, launch_k(global_avgpool_kernel, dim3((unsigned) ((warps * 32 + 255) / 256)), dim3(256), 0, ctx->stream, vi, vo), "global_avgpool_kernel");
    }
    const long long total = (long long) out->n * out->h * out->w * (out->cp >> 3);
    const dim3 grid((unsigned) ((total + 255) / 256));
    cudaError_t e;
    if (k == 2) e = launch_k(pool_kernel<2>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0);
    else if (k == 3) e = launch_k(pool_kernel<3>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0);
    else e = launch_k(pool_kernel<0>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0);
    return launch_done(ctx, e, "pool_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// Elementwise family, one thread = one 8-channel vector:
//   add + act (vk_add.comp:41-90), BatchNormalization + act (vk_batchnorm.comp:54-69), activation
//   (vk_activation.comp:41-85).
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) add_kernel(TV a, TV b, TV out, int act, float alpha) {
    pdl_wait();
    const size_t total = (size_t) out.N * out.H * out.W * (out.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG = out.Cp >> 3;
    const int c  = (int) (gid % CG) * 8;
    float x[8], y[8];
    load8(a.hi, a.lo, gid * 8, x);
    load8(b.hi, b.lo, gid * 8, y);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = (c + j < out.C) ? apply_act(x[j] + y[j], act, alpha) : 0.0f;
    store8(out.hi, out.lo, gid * 8, x);
}

// BN exactly in the shader's order: s = max(sqrt(var + 1e-3), 1e-4); y = (gamma/s)*(x - mean) + beta.
// mode 0: BN (scale = gamma/s precomputed on host as `gamma`), mode 1: activation only.
__global__ void __launch_bounds__(256) chanwise_kernel(TV in, TV out, const float* __restrict__ scale, const float* __restrict__ mean,
                                                         const float* __restrict__ beta, int mode, int act, float alpha) {
    pdl_wait();
    const size_t total = (size_t) out.N * out.H * out.W * (out.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG = out.Cp >> 3;
    const int c  = (int) (gid % CG) * 8;
    float x[8];
    load8(in.hi, in.lo, gid * 8, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float v = x[j];
        if (mode == 0) v = (__ldg(scale + c + j) * (v - __ldg(mean + c + j))) + __ldg(beta + c + j);
        x[j] = (c + j < out.C) ? apply_act(v, act, alpha) : 0.0f;
    }
    store8(out.hi, out.lo, gid * 8, x);
}

static unsigned vec_blocks(const snnb_tensor* t, int threads) {
    const size_t total = t->pixels() * (size_t) (t->cp >> 3);
    return (unsigned) ((total + threads - 1) / threads);
}

int launch_add(snnb_context* ctx, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out, int act, float alpha) {
    ctx->last_kernel = "add_kernel";
    return launch_done(ctx, launch_k(add_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(a), view(b), view(out), act, alpha), "add_kernel");
}
int launch_batchnorm(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, const snnb_weights* w, int act, float alpha) {
    return launch_done(ctx, launch_k(chanwise_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(in), view(out), w->var /* = BN scale, see pack.cpp */, w->mean, w->beta, 0, act, alpha), "chanwise_kernel");
}
int launch_activation(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, int act, float alpha) {
    return launch_done(ctx, launch_k(chanwise_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(in), view(out), nullptr, nullptr, nullptr, 1, act, alpha), "chanwise_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// Softmax over channels, per pixel (cpulayer.h:175-191: max-subtracted, fp32). One warp per pixel.
// Argmax over channels per image -> 0-based index of the FIRST maximum (core.cpp:228-233 adds 1 at the API).
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) softmax_kernel(TV in, TV out) {
    pdl_wait();
    const long long px = ((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane     = threadIdx.x & 31;
    if (px >= (long long) in.N * in.H * in.W) return;
    const size_t base = (size_t) px * in.Cp;
    float mx = -3.402823466e+38f;
    for (int c = lane; c < in.C; c += 32) mx = fmaxf(mx, load1(in.hi, in.lo, base + c));
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.0f;
    for (int c = lane; c < in.C; c += 32) sum += expf(load1(in.hi, in.lo, base + c) - mx);
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    for (int c = lane; c < out.Cp; c += 32) {
        float v = (c < in.C) ? expf(load1(in.hi, in.lo, base + c) - mx) / sum : 0.0f;
        store1(out.hi, out.lo, (size_t) px * out.Cp + c, v);
    }
}
int launch_softmax(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out) {
    const long long px = (long long) in->pixels();
    return launch_done(ctx, launch_k(softmax_kernel, dim3((unsigned) ((px * 32 + 127) / 128)), dim3(128), 0, ctx->stream, view(in), view(out)), "softmax_kernel");
}

__global__ void __launch_bounds__(128) argmax_kernel(TV in, int* __restrict__ idx) {
    pdl_wait();
    const int n    = (int) (((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= in.N) return;
    const size_t base = (size_t) n * in.H * in.W * in.Cp;
    float best = -3.402823466e+38f;
    int bi     = 0x7fffffff;
    for (int c = lane; c < in.C; c += 32) {
        float v = load1(in.hi, in.lo, base + c);
        if (v > best) best = v, bi = c;
    }
    for (int o = 16; o > 0; o >>= 1) {
        float ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi   = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) best = ob, bi = oi;
    }
    if (lane == 0) idx[n] = bi;
}
// Classifier result in one launch: fp32 values of a 1x1xC tensor and/or the arg-max per image, written wherever the pointers point -
// the streaming path hands in MAPPED PINNED HOST memory, so a small result needs no device->host copy commands at all.
__global__ void __launch_bounds__(128) result_small_kernel(TV in, float* __restrict__ values, int* __restrict__ idx) {
    pdl_wait();
    const int n    = (int) (((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= in.N) return;
    const size_t base = (size_t) n * in.Cp; // H = W = 1
    float best = -3.402823466e+38f;
    int bi     = 0x7fffffff;
    for (int c = lane; c < in.C; c += 32) {
        const float v = load1(in.hi, in.lo, base + c);
        if (values) values[(size_t) n * in.C + c] = v;
        if (v > best) best = v, bi = c;
    }
    if (!idx) return;
    for (int o = 16; o > 0; o >>= 1) { // same order as argmax_kernel: the larger value, on ties the smaller index
        float ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi   = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) best = ob, bi = oi;
    }
    if (lane == 0) idx[n] = bi;
}
int launch_result_small(snnb_context* ctx, const snnb_tensor* in, float* values, int* idx) {
    SNNB_REQUIRE(in->h == 1 && in->w == 1, "launch_result_small: a 1x1 tensor is expected");
    return launch_done(ctx, launch_k(result_small_kernel, dim3((unsigned) (((long long) in->n * 32 + 127) / 128)), dim3(128), 0, ctx->stream, view(in), values, idx), "result_small_kernel");
}
int launch_argmax(snnb_context* ctx, const snnb_tensor* in, int* dev_idx) {
    return launch_done(ctx, launch_k(argmax_kernel, dim3((unsigned) (((long long) in->n * 32 + 127) / 128)), dim3(128), 0, ctx->stream, view(in), dev_idx), "argmax_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// YOLO decode, device part (yololayer.cpp:115-164): threshold + compaction. One thread per (image, head, cell, anchor) reads the
// six values of its box and evaluates the reference's score formula; cells that could pass the confidence threshold (0.35,
// tested with a safety margin: the HOST re-evaluates the exact std::exp formula and applies the real threshold) append
// {image, scan index, d0..d5} to the batch's candidate list. The host then sorts the few survivors by scan index - the order the
// reference's loops visit them - and runs score-sort + NMS exactly as before: the detection list is bit-identical to the
// all-host decode while 16 images x 2535 cells x 18 floats no longer cross PCIe.
// ------------------------------------------------------------------------------------------------------------
__global__ void yolo_candidates_kernel(TV h0, TV h1, float thresh, int maxc, int* counts, float* cand) {
    pdl_wait();
    const int cells0 = h0.H * h0.W * 3, cells1 = h1.H * h1.W * 3;
    const long long total = (long long) h0.N * (cells0 + cells1);
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int n = (int) (gid / (cells0 + cells1)), r = (int) (gid % (cells0 + cells1));
    const bool second = r >= cells0;
    const TV& t       = second ? h1 : h0;
    const int rr = second ? r - cells0 : r, gc = rr % 3, cell = rr / 3;
    const size_t base = ((size_t) n * t.H * t.W + cell) * t.Cp + gc * 6;
    float d[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) d[i] = load1(t.hi, t.lo, base + i);
    const float prob = 1.f / ((1.f + expf(-d[4]) * (1.f + expf(-d[5])))); // yololayer.cpp:136, as parenthesised; one class: maxLogit = d[5]
    if (prob > thresh) {
        const int slot = atomicAdd(counts, 1); // ONE list for the whole batch: the host copies its head, not N fixed-size lists
        if (slot < maxc) {
            float* o = cand + (size_t) slot * 8;
            o[0]     = __int_as_float(n);
            o[1]     = __int_as_float(r); // scan index: (head, gy, gx, gc) in the reference's loop order
#pragma unroll
            for (int i = 0; i < 6; ++i) o[2 + i] = d[i];
        }
    }
}
int launch_yolo_candidates(snnb_context* ctx, const snnb_tensor* h0, const snnb_tensor* h1, float thresh, int maxc, int* counts, float* cand) {
    SNNB_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int), ctx->stream));
    const long long total = (long long) h0->n * ((long long) h0->h * h0->w + (long long) h1->h * h1->w) * 3;
    return launch_done(ctx, launch_k(yolo_candidates_kernel, dim3((unsigned) ((total + 255) / 256)), dim3(256), 0, ctx->stream, view(h0), view(h1), thresh, maxc, counts, cand), "yolo_candidates_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// Layout ops (scalar-per-element kernels: rarely on the hot path).
// ------------------------------------------------------------------------------------------------------------
// Flatten, HWC order (cpulayer.h:94-115): out[n, (y*W + x)*C + c] = in[n,y,x,c]
__global__ void flatten_kernel(TV in, TV out) {
    pdl_wait();
    const size_t total = (size_t) out.N * out.Cp;
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int n = (int) (gid / out.Cp), f = (int) (gid % out.Cp);
    float v = 0.0f;
    if (f < out.C) {
        const int c = f % in.C, px = f / in.C;
        v = load1(in.hi, in.lo, ((size_t) n * in.H * in.W + px) * in.Cp + c);
    }
    store1(out.hi, out.lo, gid, v);
}
int launch_flatten(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out) {
    const size_t total = (size_t) out->n * out->cp;
    return launch_done(ctx, launch_k(flatten_kernel, dim3((unsigned) ((total + 255) / 256)), dim3(256), 0, ctx->stream, view(in), view(out)), "flatten_kernel");
}

// Concatenate along channels (vk_concat.comp:39-52).
__global__ void concat_kernel(TV a, TV b, TV out) {
    pdl_wait();
    const size_t total = (size_t) out.N * out.H * out.W * out.Cp;
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const size_t px = gid / out.Cp;
    const int c     = (int) (gid % out.Cp);
    float v = 0.0f;
    if (c < a.C)
        v = load1(a.hi, a.lo, px * a.Cp + c);
    else if (c < a.C + b.C)
        v = load1(b.hi, b.lo, px * b.Cp + (c - a.C));
    store1(out.hi, out.lo, gid, v);
}
int launch_concat(snnb_context* ctx, const snnb_tensor* a, const snnb_tensor* b, snnb_tensor* out) {
    const size_t total = out->pixels() * out->cp;
    return launch_done(ctx, launch_k(concat_kernel, dim3((unsigned) ((total + 255) / 256)), dim3(256), 0, ctx->stream, view(a), view(b), view(out)), "concat_kernel");
}

// UpSampling2D (vk_upsampling2d_nearest.comp:43-64; vk_upsampling2d_bilinear.comp:43-86), 8-channel vectors.
__global__ void upsample_kernel(TV in, TV out, float inv, int bilinear) {
    pdl_wait();
    const int CG          = out.Cp >> 3;
    const long long total = (long long) out.N * out.H * out.W * CG;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int c  = (int) (gid % CG) * 8;
    long long r  = gid / CG;
    const int ox = (int) (r % out.W);
    r /= out.W;
    const int oy = (int) (r % out.H);
    const int n  = (int) (r / out.H);
    float v[8];
    if (!bilinear) {
        const int x1 = min(max((int) floorf((float) ox * inv), 0), in.W - 1);
        const int y1 = min(max((int) floorf((float) oy * inv), 0), in.H - 1);
        load8(in.hi, in.lo, (((size_t) n * in.H + y1) * in.W + x1) * in.Cp + c, v);
    } else {
        const float offs = 0.5f - 0.5f * inv;
        const float sx   = fminf(fmaxf((float) ox * inv - offs, 0.0f), (float) (in.W - 1));
        const float sy   = fminf(fmaxf((float) oy * inv - offs, 0.0f), (float) (in.H - 1));
        const int x11 = (int) floorf(sx), x12 = x11 + 1, y11 = (int) floorf(sy), y12 = y11 + 1;
        const float w1 = ((float) x12 - sx) * ((float) y12 - sy), w2 = (sx - (float) x11) * ((float) y12 - sy);
        const float w3 = (sx - (float) x11) * (sy - (float) y11), w4 = ((float) x12 - sx) * (sy - (float) y11);
        float t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.0f;
        auto tap = [&](int xx, int yy, float wgt) {
            if (xx < 0 || xx >= in.W || yy < 0 || yy >= in.H) return; // out-of-range texel reads 0
            load8(in.hi, in.lo, (((size_t) n * in.H + yy) * in.W + xx) * in.Cp + c, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += t[j] * wgt;
        };
        tap(x11, y11, w1);
        tap(x12, y11, w2);
        tap(x12, y12, w3);
        tap(x11, y12, w4);
    }
    store8(out.hi, out.lo, (((size_t) n * out.H + oy) * out.W + ox) * out.Cp + c, v);
}
int launch_upsample(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, float scale, bool bilinear) {
    ctx->last_kernel = "upsample_kernel";
    return launch_done(ctx, launch_k(upsample_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(in), view(out), 1.0f / scale, bilinear ? 1 : 0), "upsample_kernel");
}

// Pad (vk_pad.comp:42-70): constant(0) / replicate / reflect.
__global__ void pad_kernel(TV in, TV out, int pad_x, int pad_y, int mode) {
    pdl_wait();
    const int CG          = out.Cp >> 3;
    const long long total = (long long) out.N * out.H * out.W * CG;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int c  = (int) (gid % CG) * 8;
    long long r  = gid / CG;
    const int ox = (int) (r % out.W);
    r /= out.W;
    const int oy = (int) (r % out.H);
    const int n  = (int) (r / out.H);
    const int sx = src_coord(ox - pad_x, in.W, mode), sy = src_coord(oy - pad_y, in.H, mode);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 0.0f;
    if (sx >= 0 && sy >= 0) load8(in.hi, in.lo, (((size_t) n * in.H + sy) * in.W + sx) * in.Cp + c, v);
    store8(out.hi, out.lo, (((size_t) n * out.H + oy) * out.W + ox) * out.Cp + c, v);
}
int launch_pad(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, int pad_x, int pad_y, int mode) {
    ctx->last_kernel = "pad_kernel";
    return launch_done(ctx, launch_k(pad_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(in), view(out), pad_x, pad_y, mode), "pad_kernel");
}

// InstanceNorm (+act) (vk_instancenorm.comp:53-175): per (n, c) mean and biased variance over H*W, eps 1e-5.
// Pass 1 (instnorm_partial_kernel): grid (n x 8-channel group, spatial chunk) so that even an 8-image batch with 32 channels
// fills the GPU (the first version ran one CTA per (n, group): 32 CTAs, 500 GB/s). Each CTA reduces sum(x - K) and
// sum((x - K)^2) of its pixel range with K = the image's first pixel (shifted data: no catastrophic cancellation, one read of
// the input instead of two) through a fixed-shape tree. Pass 2 (instnorm_finalize_kernel): one thread per (n, c) adds the
// chunk partials in chunk order (deterministic) -> (mean, rstd). Pass 3: elementwise normalise + act.
__global__ void __launch_bounds__(256) instnorm_partial_kernel(TV in, float* __restrict__ partial, int chunks, int chunk_px) {
    pdl_wait();
    __shared__ float red[8][16]; // [warp][sum(x-K) x8 | sum((x-K)^2) x8]
    const int CG = in.Cp >> 3;
    const int n = blockIdx.x / CG, cg = blockIdx.x % CG, c = cg * 8;
    const int HW   = in.H * in.W;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int px0 = blockIdx.y * chunk_px, px1 = min(HW, px0 + chunk_px);
    float K[8];
    load8(in.hi, in.lo, (size_t) n * HW * in.Cp + c, K);
    float a1[8], a2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a1[j] = 0.0f, a2[j] = 0.0f;
    for (int px = px0 + threadIdx.x; px < px1; px += 256) {
        float v[8];
        load8(in.hi, in.lo, ((size_t) n * HW + px) * in.Cp + c, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float d = v[j] - K[j];
            a1[j] += d;
            a2[j] = fmaf(d, d, a2[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        for (int o = 16; o > 0; o >>= 1) a1[j] += __shfl_xor_sync(0xffffffffu, a1[j], o), a2[j] += __shfl_xor_sync(0xffffffffu, a2[j], o);
        if (lane == 0) red[warp][j] = a1[j], red[warp][8 + j] = a2[j];
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        float s = 0.0f;
        for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
        partial[(((size_t) n * CG + cg) * chunks + blockIdx.y) * 16 + threadIdx.x] = s;
    }
}
__global__ void __launch_bounds__(128) instnorm_finalize_kernel(TV in, const float* __restrict__ partial, float* __restrict__ stats, int chunks) {
    pdl_wait();
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= in.N * in.Cp) return;
    const int n = gid / in.Cp, c = gid % in.Cp, CG = in.Cp >> 3;
    const float HW = (float) (in.H * in.W);
    const float K  = load1(in.hi, in.lo, (size_t) n * in.H * in.W * in.Cp + c);
    const float* p = partial + ((size_t) n * CG + (c >> 3)) * chunks * 16 + (c & 7);
    float s1 = 0.0f, s2 = 0.0f;
    for (int k = 0; k < chunks; ++k) s1 += p[k * 16], s2 += p[k * 16 + 8];
    const float m   = s1 / HW;
    const float var = fmaxf(s2 / HW - m * m, 0.0f);
    stats[(size_t) gid * 2 + 0] = K + m;
    stats[(size_t) gid * 2 + 1] = 1.0f / sqrtf(var + 0.00001f);
}
__global__ void __launch_bounds__(256) instnorm_apply_kernel(TV in, TV out, const float* __restrict__ stats, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, int act, float alpha) {
    pdl_wait();
    const int CG          = out.Cp >> 3;
    const long long total = (long long) out.N * out.H * out.W * CG;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int c = (int) (gid % CG) * 8;
    const int n = (int) (gid / ((long long) out.H * out.W * CG));
    float v[8];
    load8(in.hi, in.lo, (size_t) gid * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float mean = stats[((size_t) n * in.Cp + c + j) * 2], rstd = stats[((size_t) n * in.Cp + c + j) * 2 + 1];
        const float mul = __ldg(gamma + c + j) * rstd;
        v[j]            = (c + j < out.C) ? apply_act((v[j] - mean) * mul + __ldg(beta + c + j), act, alpha) : 0.0f;
    }
    store8(out.hi, out.lo, (size_t) gid * 8, v);
}
int launch_instancenorm(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, const snnb_weights* w, int act, float alpha, float* scratch) {
    ctx->last_kernel = "instnorm_kernels";
    // scratch: instnorm_scratch_floats(n, cp) floats = (mean, rstd) per (n, c) + the chunk partials; the engine passes a
    // model-owned buffer (stable under CUDA graphs)
    float* stats = scratch;
    if (!stats) {
        if (ensure_stage(ctx, instnorm_scratch_floats(in->n, in->cp) * sizeof(float))) return 1;
        stats = ctx->stage_dev;
    }
    float* partial = stats + (size_t) in->n * in->cp * 2;
    const int groups = in->n * (in->cp >> 3), HW = in->h * in->w;
    int chunks = std::min(INSTNORM_MAX_CHUNKS, std::max(1, (4 * ctx->sm_count + groups - 1) / groups));
    chunks     = std::max(1, std::min(chunks, (HW + 2047) / 2048)); // at least ~2 k pixels per CTA
    const int chunk_px = (HW + chunks - 1) / chunks;
    chunks             = (HW + chunk_px - 1) / chunk_px;
    if (launch_done(ctx, launch_k(instnorm_partial_kernel, dim3((unsigned) groups, (unsigned) chunks), dim3(256), 0, ctx->stream, view(in), partial, chunks, chunk_px), "instnorm_partial_kernel")) return 1;
    if (launch_done(ctx, launch_k(instnorm_finalize_kernel, dim3((unsigned) ((in->n * in->cp + 127) / 128)), dim3(128), 0, ctx->stream, view(in), (const float*) partial, stats, chunks), "instnorm_finalize_kernel")) return 1;
    return launch_done(ctx, launch_k(instnorm_apply_kernel, dim3(vec_blocks(out, 256)), dim3(256), 0, ctx->stream, view(in), view(out), stats, w->gamma, w->beta, act, alpha), "instnorm_apply_kernel");
}

// Subpixel: depth_to_space(r) + tanh (vk_subpixel.comp:43-70; component = x%r + r*(y%r), fs_subpixel.glsl:41).
__global__ void subpixel_kernel(TV in, TV out, int r) {
    pdl_wait();
    const long long total = (long long) out.N * out.H * out.W;
    const long long gid   = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int ox = (int) (gid % out.W);
    long long q  = gid / out.W;
    const int oy = (int) (q % out.H);
    const int n  = (int) (q / out.H);
    const int comp = (ox % r) + r * (oy % r);
    const float v  = load1(in.hi, in.lo, (((size_t) n * in.H + oy / r) * in.W + ox / r) * in.Cp + comp);
    float o[8];
    o[0] = tanhf(v);
#pragma unroll
    for (int j = 1; j < 8; ++j) o[j] = 0.0f;
    store8(out.hi, out.lo, (size_t) gid * out.Cp, o); // out.C == 1, Cp == 8
}
int launch_subpixel(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* out, int r) {
    const long long total = (long long) out->pixels();
    return launch_done(ctx, launch_k(subpixel_kernel, dim3((unsigned) ((total + 255) / 256)), dim3(256), 0, ctx->stream, view(in), view(out), r), "subpixel_kernel");
}

// ------------------------------------------------------------------------------------------------------------
// API edge: fp32 NHWC (dense pitch C) <-> split-fp16 (pitch Cp).
// ------------------------------------------------------------------------------------------------------------
__global__ void split_kernel(const float* __restrict__ src, TV t, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (c + j < t.C) ? __ldg(src + px * t.C + c + j) : 0.0f;
    if (!f.only) store8(t.hi, t.lo, gid * 8, v);
    if (f.hi) store_feed(f, px, t.H, t.W, v);
}
// u8 image (dense pitch C) -> (x - mean[c]) * norm[c] -> split-fp16: the reference's convertToRGBA32FAndNormalize
// (core/inc/snn/imageTexture.h:114) done on the device, so only a quarter of the fp32 bytes cross PCIe.
struct U8Norm {
    float mean[4], norm[4];
};
__global__ void split_u8_kernel(const uint8_t* __restrict__ src, TV t, U8Norm q, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (c + j < t.C) ? ((float) __ldg(src + px * t.C + c + j) - q.mean[(c + j) & 3]) * q.norm[(c + j) & 3] : 0.0f;
    if (!f.only) store8(t.hi, t.lo, gid * 8, v);
    if (f.hi) store_feed(f, px, t.H, t.W, v);
}
__global__ void merge_kernel(TV t, float* __restrict__ dst, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    float v[8];
    if (f.only) load_feed(f, px, t.H, t.W, v); // C <= 4: one vector per pixel
    else load8(t.hi, t.lo, gid * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (c + j < t.C) dst[px * t.C + c + j] = v[j];
}
int launch_split_f32(snnb_context* ctx, const float* dev_nhwc, snnb_tensor* t) {
    return launch_done(ctx, launch_k(split_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, dev_nhwc, view(t), feed_view(t)), "split_kernel");
}
int launch_split_u8(snnb_context* ctx, const uint8_t* dev_nhwc_u8, snnb_tensor* t, const float mean[4], const float norm[4]) {
    U8Norm q;
    for (int i = 0; i < 4; ++i) q.mean[i] = mean[i], q.norm[i] = norm[i];
    return launch_done(ctx, launch_k(split_u8_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, dev_nhwc_u8, view(t), q, feed_view(t)), "split_u8_kernel");
}
// u8 image of ANOTHER size -> resize (linear or nearest) -> (x - mean[c]) * norm[c] -> split-fp16: ImageTexture::resize
// (core/inc/snn/imageTexture.h:137) = shadertemplate_vk_resize.comp:42-61: the output texel centre (x + 0.5) / outW is sampled from
// the source texture with the sampler's filter (texel centres at (i + 0.5) / inW, clamp to edge), then normalised.
__global__ void resize_u8_kernel(const uint8_t* __restrict__ src, int sh, int sw, TV t, U8Norm q, int linear, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    const int ox = (int) (px % t.W), oy = (int) ((px / t.W) % t.H), n = (int) (px / ((size_t) t.W * t.H));
    const float fx = ((float) ox + 0.5f) / (float) t.W * (float) sw, fy = ((float) oy + 0.5f) / (float) t.H * (float) sh;
    const uint8_t* img = src + (size_t) n * sh * sw * t.C;
    float v[8];
    if (linear) {
        const float sx = fx - 0.5f, sy = fy - 0.5f;
        const float x0f = floorf(sx), y0f = floorf(sy);
        const float ax = sx - x0f, ay = sy - y0f;
        const int x0 = min(max((int) x0f, 0), sw - 1), x1 = min(max((int) x0f + 1, 0), sw - 1);
        const int y0 = min(max((int) y0f, 0), sh - 1), y1 = min(max((int) y0f + 1, 0), sh - 1);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float r = 0.0f;
            if (c + j < t.C) {
                const float p00 = (float) __ldg(img + ((size_t) y0 * sw + x0) * t.C + c + j), p01 = (float) __ldg(img + ((size_t) y0 * sw + x1) * t.C + c + j);
                const float p10 = (float) __ldg(img + ((size_t) y1 * sw + x0) * t.C + c + j), p11 = (float) __ldg(img + ((size_t) y1 * sw + x1) * t.C + c + j);
                const float top = p00 + ax * (p01 - p00), bot = p10 + ax * (p11 - p10);
                r               = ((top + ay * (bot - top)) - q.mean[(c + j) & 3]) * q.norm[(c + j) & 3];
            }
            v[j] = r;
        }
    } else {
        const int x0 = min((int) fx, sw - 1), y0 = min((int) fy, sh - 1);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (c + j < t.C) ? ((float) __ldg(img + ((size_t) y0 * sw + x0) * t.C + c + j) - q.mean[(c + j) & 3]) * q.norm[(c + j) & 3] : 0.0f;
    }
    if (!f.only) store8(t.hi, t.lo, gid * 8, v);
    if (f.hi) store_feed(f, px, t.H, t.W, v);
}
int launch_resize_u8(snnb_context* ctx, const uint8_t* dev_nhwc_u8, int src_h, int src_w, snnb_tensor* t, const float mean[4], const float norm[4], bool linear) {
    U8Norm q;
    for (int i = 0; i < 4; ++i) q.mean[i] = mean[i], q.norm[i] = norm[i];
    return launch_done(ctx, launch_k(resize_u8_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, dev_nhwc_u8, src_h, src_w, view(t), q, linear ? 1 : 0, feed_view(t)), "resize_u8_kernel");
}
// tensor -> 8-bit image, dense NHWC: clamp(round(v * scale + offset), 0, 255) (the image-to-image models' outputs: style transfer,
// super-resolution); a quarter of the fp32 bytes cross PCIe on the way back
__global__ void merge_u8_kernel(TV t, uint8_t* __restrict__ dst, float scale, float offset) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    float v[8];
    load8(t.hi, t.lo, gid * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (c + j < t.C) dst[px * t.C + c + j] = (uint8_t) fminf(fmaxf(rintf(v[j] * scale + offset), 0.0f), 255.0f);
}
int launch_merge_u8(snnb_context* ctx, const snnb_tensor* t, uint8_t* dev_nhwc_u8, float scale, float offset) {
    return launch_done(ctx, launch_k(merge_u8_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, view(t), dev_nhwc_u8, scale, offset), "merge_u8_kernel");
}
int launch_merge_f32(snnb_context* ctx, const snnb_tensor* t, float* dev_nhwc) {
    return launch_done(ctx, launch_k(merge_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, view(t), dev_nhwc, feed_view(t)), "merge_kernel");
}

} // namespace snnb
