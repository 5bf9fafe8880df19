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
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

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
    const int variant[6] = {CONV_SIMT, 0, 0, 1, 0, 0}; // fp32 FMAs on the folded fp32 weights: no product form
    std::copy(variant, variant + 6, ctx->last_conv);
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
        static_assert(TX == 4, "the launch names below spell TX");
        if (a.stride == 1) return launch_done(ctx, launch_k(depthwise_kernel<3, 1, TX>, dim3(blocks), dim3(128), 0, ctx->stream, p), "depthwise_kernel<3, 1, 4>");
        return launch_done(ctx, launch_k(depthwise_kernel<3, 2, TX>, dim3(blocks), dim3(128), 0, ctx->stream, p), "depthwise_kernel<3, 2, 4>");
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

int gap_dense_parts(int in_c, int out_c) {
    const int icp = round_up(in_c, 8), ocp = round_up(out_c, 8);
    int parts = std::max(1, std::min(GD_THREADS / (icp >> 3), 8));
    while (parts > 1 && (size_t) (parts * icp + (GD_THREADS / 32 + 1) * ocp) * sizeof(float) > 48 * 1024) --parts;
    return (size_t) (parts * icp + (GD_THREADS / 32 + 1) * ocp) * sizeof(float) > 48 * 1024 ? 0 : parts;
}
static int gap_dense_parts(const snnb_tensor* in, const snnb_tensor* out) { return gap_dense_parts(in->cp, out->cp); }
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
    if (k == 2) return launch_done(ctx, launch_k(pool_kernel<2>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0), "pool_kernel<2>");
    if (k == 3) return launch_done(ctx, launch_k(pool_kernel<3>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0), "pool_kernel<3>");
    return launch_done(ctx, launch_k(pool_kernel<0>, grid, dim3(256), 0, ctx->stream, vi, vo, k, stride, avg ? 1 : 0), "pool_kernel<0>");
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
// Argmax over channels per image -> index of the FIRST maximum plus base_index (0 where the host adds 1 at the API,
// core.cpp:228-233; 1 where the 1-based classes stay in device memory). NaN scores: argmax_take below.
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

// The index is std::max_element's (the reference's core.cpp:230-232) for every input, NaN included: 0 when score 0 is NaN (no score
// compares above it) or when no score is a number; otherwise the first maximum of the scores that are numbers (a later NaN never
// compares above the running maximum). So the index is always in [0, C) and the + 1 of the 1-based classes cannot overflow.
// A lane scans channels lane, lane + 32, ... in order; ARGMAX_NONE marks a lane that has seen no number yet.
constexpr int ARGMAX_NONE = 0x7fffffff;
__device__ __forceinline__ void argmax_take(float& best, int& bi, float v, int c) {
    if (v == v && (bi == ARGMAX_NONE || v > best)) best = v, bi = c;
}
// The warp's first maximum from the lanes' (best, bi): the larger value, on ties the smaller index; lanes without a number lose.
// lane 0 returns the image's index, nan0: score 0 is NaN.
__device__ __forceinline__ int argmax_warp(float best, int bi, bool nan0) {
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi   = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi != ARGMAX_NONE && (bi == ARGMAX_NONE || ob > best || (ob == best && oi < bi))) best = ob, bi = oi;
    }
    return (nan0 || bi == ARGMAX_NONE) ? 0 : bi;
}
__global__ void __launch_bounds__(128) argmax_kernel(TV in, int* __restrict__ idx, int base_index) {
    pdl_wait();
    const int n    = (int) (((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= in.N) return;
    const size_t base = (size_t) n * in.H * in.W * in.Cp;
    float best = 0.0f;
    int bi     = ARGMAX_NONE;
    bool nan0  = false;
    for (int c = lane; c < in.C; c += 32) {
        const float v = load1(in.hi, in.lo, base + c);
        if (c == 0) nan0 = v != v;
        argmax_take(best, bi, v, c);
    }
    const int i = argmax_warp(best, bi, nan0);
    if (lane == 0) idx[n] = i + base_index;
}
// Classifier result in one launch: fp32 values of a 1x1xC tensor and/or the arg-max per image, written wherever the pointers point -
// the streaming path hands in MAPPED PINNED HOST memory, so a small result needs no device->host copy commands at all.
__global__ void __launch_bounds__(128) result_small_kernel(TV in, float* __restrict__ values, int* __restrict__ idx) {
    pdl_wait();
    const int n    = (int) (((long long) blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= in.N) return;
    const size_t base = (size_t) n * in.Cp; // H = W = 1
    float best = 0.0f;
    int bi     = ARGMAX_NONE;
    bool nan0  = false;
    for (int c = lane; c < in.C; c += 32) {
        const float v = load1(in.hi, in.lo, base + c);
        if (values) values[(size_t) n * in.C + c] = v;
        if (c == 0) nan0 = v != v;
        argmax_take(best, bi, v, c);
    }
    if (!idx) return;
    const int i = argmax_warp(best, bi, nan0); // argmax_kernel's scan and reduction, so the two agree on every input
    if (lane == 0) idx[n] = i;
}
int launch_result_small(snnb_context* ctx, const snnb_tensor* in, float* values, int* idx) {
    SNNB_REQUIRE(in->h == 1 && in->w == 1, "launch_result_small: a 1x1 tensor is expected");
    return launch_done(ctx, launch_k(result_small_kernel, dim3((unsigned) (((long long) in->n * 32 + 127) / 128)), dim3(128), 0, ctx->stream, view(in), values, idx), "result_small_kernel");
}
int launch_argmax(snnb_context* ctx, const snnb_tensor* in, int* dev_idx, int base_index) {
    return launch_done(ctx, launch_k(argmax_kernel, dim3((unsigned) (((long long) in->n * 32 + 127) / 128)), dim3(128), 0, ctx->stream, view(in), dev_idx, base_index),
                       "argmax_kernel");
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
// YOLO decode, all on the device (snnb_model_detect_device): exact threshold, stable score sort, greedy NMS per image. The host
// counterpart is YOLOLayer::decode + nms (layers.cpp: decodeCell, iou, nms; yololayer.cpp:56-164). Arithmetic contract:
//   - exp is the correctly rounded float exponential, (float) exp((double) x). The host's std::exp (glibc expf) is not correctly
//     rounded for every input, so a score or box can differ from the host's by the ulp or so that one exp differs.
//   - every + - * / is an IEEE-rounded intrinsic, so nvcc cannot contract a product and a sum into an FMA; the host build has no
//     FMA either. Each operation is the host's, in the host's order.
// Three kernels, one list per image: yolo_select_kernel evaluates every cell and appends a 64-bit key for each one that passes;
// yolo_rank_kernel sorts the keys by rank; yolo_nms_kernel decodes the boxes in that order and suppresses greedily.
// ------------------------------------------------------------------------------------------------------------
namespace yolo_dev { // layers.cpp: kGridScale, kAnchors, kMasks, GC, NFIX, ONUM, kConfThresh, kIouThresh (yololayer.cpp:31-38, 182-183)
__constant__ int kGridScale[2] = {32, 16};
__constant__ float kAnchors[12] = {10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319};
__constant__ float kMasks[6]    = {3, 4, 5, 1, 2, 3};
constexpr int GC = 3, NFIX = 5, ONUM = 6;
constexpr float kConfThresh = 0.35f, kIouThresh = 0.45f;
constexpr int NMS_THREADS = 128; // candidates resolved per step of yolo_nms_kernel: a 128-bit suppression mask (two words) each
constexpr int MAX_ROWS    = 100; // snnb_model_get_boxes returns at most 100 rows per image
}

struct YoloBox {
    int cls;
    float score, x, y, w, h;
};
__device__ __forceinline__ float exp_cr(float x) { return (float) exp((double) x); }

// decodeCell (layers.cpp) for the cell at `scan` of image n: scan = (head, gy, gx, gc) in the order the host's loops visit the cells.
// Returns false below the confidence threshold; otherwise out.score is set, and the rest of the box when `box` is set.
__device__ bool yolo_decode_cell(const TV& h0, const TV& h1, int n, int scan, bool box, YoloBox& out) {
    using namespace yolo_dev;
    const int cells0 = h0.H * h0.W * GC;
    const int yi     = scan >= cells0 ? 1 : 0;
    const TV& t      = yi ? h1 : h0;
    const int s = yi ? scan - cells0 : scan, gc = s % GC, cell = s / GC;
    const int gw = t.W, gh = t.H, gx = cell % gw, gy = cell / gw;
    const size_t base = ((size_t) n * gh * gw + cell) * t.Cp + gc * ONUM;
    float d[ONUM];
#pragma unroll
    for (int i = 0; i < ONUM; ++i) d[i] = load1(t.hi, t.lo, base + i);
    int cls        = 0;
    float maxLogit = -3.402823466e+38f;
#pragma unroll
    for (int i = NFIX; i < ONUM; ++i)
        if (d[i] > maxLogit) maxLogit = d[i], cls = i - NFIX;
    // prob = 1.f / ((1.f + exp(-d[4]) * (1.f + exp(-maxLogit))))
    const float prob = __fdiv_rn(1.f, __fadd_rn(1.f, __fmul_rn(exp_cr(-d[4]), __fadd_rn(1.f, exp_cr(-maxLogit)))));
    if (!(prob > kConfThresh)) return false;
    out.score = prob;
    if (!box) return true;
    const int ai   = (int) kMasks[gc + yi * GC];
    const float bw = kAnchors[ai * 2], bh = kAnchors[ai * 2 + 1];
    const int netW = kGridScale[yi] * gw, netH = kGridScale[yi] * gh;
    // cx = (gx + 1.0f / (1.0f + exp(-d[0]))) / gw, cy likewise; w_ = exp(d[2]) * bw / netW, h_ likewise
    const float cx = __fdiv_rn(__fadd_rn((float) gx, __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_cr(-d[0])))), (float) gw);
    const float cy = __fdiv_rn(__fadd_rn((float) gy, __fdiv_rn(1.0f, __fadd_rn(1.0f, exp_cr(-d[1])))), (float) gh);
    const float w_ = __fdiv_rn(__fmul_rn(exp_cr(d[2]), bw), (float) netW), h_ = __fdiv_rn(__fmul_rn(exp_cr(d[3]), bh), (float) netH);
    out = YoloBox {cls, prob, __fsub_rn(cx, __fdiv_rn(w_, 2.f)), __fsub_rn(cy, __fdiv_rn(h_, 2.f)), w_, h_};
    return true;
}
// iou (layers.cpp), with std::max(a, b) = a < b ? b : a and std::min(a, b) = b < a ? b : a
__device__ __forceinline__ float yolo_iou(const YoloBox& a, const YoloBox& b) {
    const float ix0 = a.x < b.x ? b.x : a.x, iy0 = a.y < b.y ? b.y : a.y;
    const float ax1 = __fadd_rn(a.x, a.w), bx1 = __fadd_rn(b.x, b.w), ay1 = __fadd_rn(a.y, a.h), by1 = __fadd_rn(b.y, b.h);
    const float ix1 = bx1 < ax1 ? bx1 : ax1, iy1 = by1 < ay1 ? by1 : ay1;
    if (ix1 < ix0 || iy1 < iy0) return 0;
    const float inter = __fmul_rn(__fsub_rn(ix1, ix0), __fsub_rn(iy1, iy0));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(__fmul_rn(a.w, a.h), __fmul_rn(b.w, b.h)), inter));
}
// Sort key: std::stable_sort by descending score over the scan-ordered list == descending (score, -scan). Scores are > 0.35, so
// their bits order like unsigned integers; every key is distinct.
__device__ __forceinline__ unsigned long long yolo_key(float score, int scan) {
    return ((unsigned long long) __float_as_uint(score) << 32) | (unsigned long long) (0xffffffffu - (unsigned) scan);
}
__device__ __forceinline__ int yolo_key_scan(unsigned long long k) { return (int) (0xffffffffu - (unsigned) (k & 0xffffffffu)); }

// One thread per (cell, anchor) of image blockIdx.y: cells that pass append their key to the image's list (arbitrary order).
__global__ void __launch_bounds__(256) yolo_select_kernel(TV h0, TV h1, int cap, int* __restrict__ counts, unsigned long long* __restrict__ keys) {
    pdl_wait();
    const int n = blockIdx.y, scan = blockIdx.x * blockDim.x + threadIdx.x;
    if (scan >= cap) return;
    YoloBox b;
    if (yolo_decode_cell(h0, h1, n, scan, false, b)) keys[(size_t) n * cap + atomicAdd(&counts[n], 1)] = yolo_key(b.score, scan);
}

// Rank sort of image blockIdx.y's keys: the rank of a key is the number of larger keys, so sorted[rank] is the descending order.
// Quadratic in the image's candidate count, spread over the grid; blocks past the count exit at once.
__global__ void __launch_bounds__(256) yolo_rank_kernel(int cap, const int* __restrict__ counts, const unsigned long long* __restrict__ keys,
                                                         unsigned long long* __restrict__ sorted) {
    pdl_wait();
    __shared__ unsigned long long tile[256];
    const int n = blockIdx.y, count = counts[n];
    if ((int) (blockIdx.x * blockDim.x) >= count) return;
    const unsigned long long* k = keys + (size_t) n * cap;
    const int i                 = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long mine = i < count ? k[i] : 0ull;
    int rank = 0;
    for (int t0 = 0; t0 < count; t0 += 256) {
        __syncthreads();
        if (t0 + (int) threadIdx.x < count) tile[threadIdx.x] = k[t0 + threadIdx.x];
        __syncthreads();
        const int m = min(256, count - t0);
        for (int j = 0; j < m; ++j) rank += tile[j] > mine ? 1 : 0;
    }
    if (i < count) sorted[(size_t) n * cap + rank] = mine;
}

// Greedy NMS of one list in descending score order, by one CTA of NMS_THREADS threads (nms, layers.cpp): a box is kept unless a kept
// box before it of the same class overlaps it with IoU > 0.45, which is what the host's loop computes. The list is walked NMS_THREADS
// candidates at a time: each thread fetches one (boxes(i, b): false when candidate i is not a box), tests it against the boxes kept so
// far and records which earlier candidates of the step would suppress it; thread 0 then resolves the step in order. The walk stops at
// max_rows kept boxes: later boxes cannot change earlier ones.
// rows[n][max_rows][6] = {class, score, x, y, w, h}, zero past the count; out_counts[n] = the number of rows. The box source is a
// template argument so that yolo_nms_kernel (cells decoded from the heads) and roi_merge_nms_kernel (boxes already decoded) share this
// step; yolo_nms_kernel's machine code is the same as before the step was lifted out of it.
template <class Boxes>
__device__ __forceinline__ void yolo_greedy_nms(const Boxes& boxes, int count, int max_rows, int n, float* __restrict__ rows, int* __restrict__ out_counts) {
    using namespace yolo_dev;
    __shared__ YoloBox kept[MAX_ROWS];
    __shared__ YoloBox step[NMS_THREADS];
    __shared__ unsigned long long mask[NMS_THREADS][2];
    __shared__ int live[NMS_THREADS];
    __shared__ int nkept;
    const int tid = threadIdx.x;
    if (tid == 0) nkept = 0;
    __syncthreads();
    for (int c0 = 0; c0 < count && nkept < max_rows; c0 += NMS_THREADS) {
        const int i = c0 + tid;
        YoloBox b {};
        bool alive = i < count;
        if (alive) alive = boxes(i, b);
        step[tid] = b;
        const int k0 = nkept;
        for (int k = 0; k < k0 && alive; ++k)
            if (kept[k].cls == b.cls && yolo_iou(kept[k], b) > kIouThresh) alive = false;
        live[tid] = alive ? 1 : 0;
        __syncthreads();
        unsigned long long m0 = 0, m1 = 0; // bit j: live candidate j of this step (j < tid) suppresses this one
        if (alive)
            for (int j = 0; j < tid; ++j)
                if (live[j] && step[j].cls == b.cls && yolo_iou(step[j], b) > kIouThresh) {
                    if (j < 64) m0 |= 1ull << j;
                    else m1 |= 1ull << (j - 64);
                }
        mask[tid][0] = m0, mask[tid][1] = m1;
        __syncthreads();
        if (tid == 0) {
            unsigned long long k0m = 0, k1m = 0; // the candidates of this step kept so far
            int nk = nkept;
            for (int j = 0; j < NMS_THREADS && nk < max_rows; ++j) {
                if (!live[j] || (mask[j][0] & k0m) || (mask[j][1] & k1m)) continue;
                if (j < 64) k0m |= 1ull << j;
                else k1m |= 1ull << (j - 64);
                kept[nk++] = step[j];
            }
            nkept = nk;
        }
        __syncthreads();
    }
    const int nk = nkept;
    float* r = rows + (size_t) n * max_rows * 6;
    for (int e = tid; e < max_rows * 6; e += NMS_THREADS) {
        const int k = e / 6, f = e % 6;
        float v = 0.0f;
        if (k < nk) {
            const YoloBox& b = kept[k];
            v = f == 0 ? (float) b.cls : f == 1 ? b.score : f == 2 ? b.x : f == 3 ? b.y : f == 4 ? b.w : b.h;
        }
        r[e] = v;
    }
    if (tid == 0) out_counts[n] = nk;
}
// Image n's candidates: the cells of its sorted keys, decoded from the heads
struct YoloCellBoxes {
    TV h0, h1;
    int n;
    const unsigned long long* s;
    __device__ __forceinline__ bool operator()(int i, YoloBox& b) const { return yolo_decode_cell(h0, h1, n, yolo_key_scan(s[i]), true, b); }
};
// Greedy NMS of image blockIdx.x over its sorted list: rows[n][max_rows][6], out_counts[n]
__global__ void __launch_bounds__(yolo_dev::NMS_THREADS) yolo_nms_kernel(TV h0, TV h1, int cap, const int* __restrict__ counts,
                                                                        const unsigned long long* __restrict__ sorted, int max_rows,
                                                                        float* __restrict__ rows, int* __restrict__ out_counts) {
    pdl_wait();
    const int n = blockIdx.x;
    yolo_greedy_nms(YoloCellBoxes {h0, h1, n, sorted + (size_t) n * cap}, counts[n], max_rows, n, rows, out_counts);
}

// scratch: the candidate count of every image (rounded up to 256 bytes), then the keys and the sorted keys, [N][cells per image] each
static size_t yolo_counts_bytes(int N) { return ((size_t) N * sizeof(int) + 255) & ~(size_t) 255; }
static long long yolo_cells(const snnb_tensor* h0, const snnb_tensor* h1) { return ((long long) h0->h * h0->w + (long long) h1->h * h1->w) * yolo_dev::GC; }
size_t yolo_detect_scratch_bytes(const snnb_tensor* h0, const snnb_tensor* h1) {
    return yolo_counts_bytes(h0->n) + (size_t) h0->n * (size_t) yolo_cells(h0, h1) * 2 * sizeof(unsigned long long);
}
int launch_yolo_detect(snnb_context* ctx, const snnb_tensor* h0, const snnb_tensor* h1, void* scratch, int max_rows, float* rows, int* out_counts) {
    SNNB_REQUIRE(h0->n == h1->n && h0->c >= yolo_dev::GC * yolo_dev::ONUM && h1->c >= yolo_dev::GC * yolo_dev::ONUM, "launch_yolo_detect: two heads of >= 18 channels");
    SNNB_REQUIRE(max_rows >= 1 && max_rows <= yolo_dev::MAX_ROWS, "launch_yolo_detect: max_rows %d is outside 1..%d", max_rows, yolo_dev::MAX_ROWS);
    const long long capl = yolo_cells(h0, h1);
    SNNB_REQUIRE(capl < 0x7fffffffLL, "launch_yolo_detect: %lld cells per image", capl);
    const int cap = (int) capl, N = h0->n;
    int* counts  = static_cast<int*>(scratch);
    auto* keys   = reinterpret_cast<unsigned long long*>(static_cast<char*>(scratch) + yolo_counts_bytes(N));
    auto* sorted = keys + (size_t) N * cap;
    SNNB_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int) * N, ctx->stream));
    const dim3 grid((unsigned) ((cap + 255) / 256), (unsigned) N);
    if (launch_done(ctx, launch_k(yolo_select_kernel, grid, dim3(256), 0, ctx->stream, view(h0), view(h1), cap, counts, keys), "yolo_select_kernel")) return 1;
    if (launch_done(ctx, launch_k(yolo_rank_kernel, grid, dim3(256), 0, ctx->stream, cap, (const int*) counts, (const unsigned long long*) keys, sorted), "yolo_rank_kernel")) return 1;
    return launch_done(ctx, launch_k(yolo_nms_kernel, dim3((unsigned) N), dim3(yolo_dev::NMS_THREADS), 0, ctx->stream, view(h0), view(h1), cap, (const int*) counts,
                                     (const unsigned long long*) sorted, max_rows, rows, out_counts),
                       "yolo_nms_kernel");
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
// ImageTexture::resize (core/inc/snn/imageTexture.h:137) = shadertemplate_vk_resize.comp:42-61: the output texel centre (x + 0.5) / outW
// is sampled from the source texture with the sampler's filter (texel centres at (i + 0.5) / inW, clamp to edge). The taps of output
// pixel (ox, oy) of a W x H image from a sw x sh source, and the bilinear blend: shared by resize_u8_kernel and frame_input_kernel, so
// that a frame is resampled exactly as an 8-bit image is. Nearest: x0 == x1, y0 == y1, and blend() is not used.
struct ResizeTaps {
    int x0, x1, y0, y1;
    float ax, ay;
    __device__ __forceinline__ float blend(float p00, float p01, float p10, float p11) const {
        const float top = p00 + ax * (p01 - p00), bot = p10 + ax * (p11 - p10);
        return top + ay * (bot - top);
    }
};
// ResizeTaps::blend with every + - * rounded on its own: nothing is contracted into an FMA, so numpy float32 restates it exactly.
__device__ __forceinline__ float blend_rn(const ResizeTaps& r, float p00, float p01, float p10, float p11) {
    const float top = __fadd_rn(p00, __fmul_rn(r.ax, __fsub_rn(p01, p00)));
    const float bot = __fadd_rn(p10, __fmul_rn(r.ax, __fsub_rn(p11, p10)));
    return __fadd_rn(top, __fmul_rn(r.ay, __fsub_rn(bot, top)));
}
// The source position of output pixel (ox, oy), then its taps.
__device__ __forceinline__ float2 resize_pos(int ox, int oy, int W, int H, int sw, int sh) {
    return make_float2(((float) ox + 0.5f) / (float) W * (float) sw, ((float) oy + 0.5f) / (float) H * (float) sh);
}
__device__ __forceinline__ ResizeTaps resize_taps(float2 pos, int sw, int sh, int linear) {
    const float fx = pos.x, fy = pos.y;
    ResizeTaps r;
    if (linear) {
        const float sx = fx - 0.5f, sy = fy - 0.5f;
        const float x0f = floorf(sx), y0f = floorf(sy);
        r.ax = sx - x0f, r.ay = sy - y0f;
        r.x0 = min(max((int) x0f, 0), sw - 1), r.x1 = min(max((int) x0f + 1, 0), sw - 1);
        r.y0 = min(max((int) y0f, 0), sh - 1), r.y1 = min(max((int) y0f + 1, 0), sh - 1);
    } else {
        r.x0 = r.x1 = min((int) fx, sw - 1), r.y0 = r.y1 = min((int) fy, sh - 1);
        r.ax = r.ay = 0.0f;
    }
    return r;
}
// u8 image of ANOTHER size -> resize (linear or nearest, resize_taps) -> (x - mean[c]) * norm[c] -> split-fp16.
__global__ void resize_u8_kernel(const uint8_t* __restrict__ src, int sh, int sw, TV t, U8Norm q, int linear, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int CG    = t.Cp >> 3;
    const size_t px = gid / CG;
    const int c     = (int) (gid % CG) * 8;
    const int ox = (int) (px % t.W), oy = (int) ((px / t.W) % t.H), n = (int) (px / ((size_t) t.W * t.H));
    const float2 pos = resize_pos(ox, oy, t.W, t.H, sw, sh);
    const uint8_t* img = src + (size_t) n * sh * sw * t.C;
    float v[8];
    if (linear) {
        const ResizeTaps r = resize_taps(pos, sw, sh, 1);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float o = 0.0f;
            if (c + j < t.C) {
                const float p00 = (float) __ldg(img + ((size_t) r.y0 * sw + r.x0) * t.C + c + j), p01 = (float) __ldg(img + ((size_t) r.y0 * sw + r.x1) * t.C + c + j);
                const float p10 = (float) __ldg(img + ((size_t) r.y1 * sw + r.x0) * t.C + c + j), p11 = (float) __ldg(img + ((size_t) r.y1 * sw + r.x1) * t.C + c + j);
                o               = (r.blend(p00, p01, p10, p11) - q.mean[(c + j) & 3]) * q.norm[(c + j) & 3];
            }
            v[j] = o;
        }
    } else {
        const ResizeTaps r = resize_taps(pos, sw, sh, 0);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (c + j < t.C) ? ((float) __ldg(img + ((size_t) r.y0 * sw + r.x0) * t.C + c + j) - q.mean[(c + j) & 3]) * q.norm[(c + j) & 3] : 0.0f;
    }
    if (!f.only) store8(t.hi, t.lo, gid * 8, v);
    if (f.hi) store_feed(f, px, t.H, t.W, v);
}
int launch_resize_u8(snnb_context* ctx, const uint8_t* dev_nhwc_u8, int src_h, int src_w, snnb_tensor* t, const float mean[4], const float norm[4], bool linear) {
    U8Norm q;
    for (int i = 0; i < 4; ++i) q.mean[i] = mean[i], q.norm[i] = norm[i];
    return launch_done(ctx, launch_k(resize_u8_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, dev_nhwc_u8, src_h, src_w, view(t), q, linear ? 1 : 0, feed_view(t)), "resize_u8_kernel");
}
// A model output value as 8 bits: clamp(round(v * scale + offset), 0, 255). Every U8 output (merge_u8_kernel, device_output_kernel<u8>,
// frame_output_kernel) quantises here, so that they cannot drift apart.
__device__ __forceinline__ float quant_u8(float v, float scale, float offset) { return fminf(fmaxf(rintf(v * scale + offset), 0.0f), 255.0f); }
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
        if (c + j < t.C) dst[px * t.C + c + j] = (uint8_t) quant_u8(v[j], scale, offset);
}
int launch_merge_u8(snnb_context* ctx, const snnb_tensor* t, uint8_t* dev_nhwc_u8, float scale, float offset) {
    return launch_done(ctx, launch_k(merge_u8_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, view(t), dev_nhwc_u8, scale, offset), "merge_u8_kernel");
}
int launch_merge_f32(snnb_context* ctx, const snnb_tensor* t, float* dev_nhwc) {
    return launch_done(ctx, launch_k(merge_kernel, dim3(vec_blocks(t, 256)), dim3(256), 0, ctx->stream, view(t), dev_nhwc, feed_view(t)), "merge_kernel");
}

// Caller-owned device buffers (snnb_model_run_device): F32 / F16 / U8, dense NHWC or NCHW. One thread per (pixel, 8-channel group) as
// in split_kernel / merge_kernel, and the same values and stores. In NCHW the pixel is the fastest-moving index, so consecutive threads
// read (write) consecutive pixels of one channel plane; their 16-byte tensor-side vectors are Cp * 2 bytes apart.
struct EdgeIndex {
    size_t px;   // linear (n, y, x) pixel
    int c;       // first channel of the group
    size_t base; // buffer element of channel 0 of this pixel
    size_t step; // buffer elements from one channel to the next
};
__device__ __forceinline__ EdgeIndex edge_index(size_t gid, const TV& t, int nchw) {
    const int CG    = t.Cp >> 3;
    const size_t HW = (size_t) t.H * t.W;
    EdgeIndex e;
    if (nchw) {
        const size_t hw = gid % HW, q = gid / HW;
        const size_t n  = q / CG;
        e.c    = (int) (q % CG) * 8;
        e.px   = n * HW + hw;
        e.base = n * t.C * HW + hw;
        e.step = HW;
    } else {
        e.px   = gid / CG;
        e.c    = (int) (gid % CG) * 8;
        e.base = e.px * t.C;
        e.step = 1;
    }
    return e;
}
__device__ __forceinline__ float edge_in(const float* p, int, const U8Norm&) { return __ldg(p); }
__device__ __forceinline__ float edge_in(const __half* p, int, const U8Norm&) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float edge_in(const uint8_t* p, int c, const U8Norm& q) { return ((float) __ldg(p) - q.mean[c & 3]) * q.norm[c & 3]; } // = split_u8_kernel
__device__ __forceinline__ void edge_out(float* p, float v, float, float) { *p = v; }
__device__ __forceinline__ void edge_out(__half* p, float v, float, float) { *p = __float2half_rn(v); }
__device__ __forceinline__ void edge_out(uint8_t* p, float v, float scale, float offset) { *p = (uint8_t) quant_u8(v, scale, offset); }

template <typename T>
__global__ void device_input_kernel(const T* __restrict__ src, int nchw, TV t, U8Norm q, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const EdgeIndex e = edge_index(gid, t, nchw);
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (e.c + j < t.C) ? edge_in(src + e.base + (size_t) (e.c + j) * e.step, e.c + j, q) : 0.0f;
    if (!f.only) store8(t.hi, t.lo, e.px * t.Cp + e.c, v);
    if (f.hi) store_feed(f, e.px, t.H, t.W, v);
}
// NCHW input with more than 8 channels: a tile of 32 pixels x 64 channels passes through shared memory, so that the reads of a channel
// plane AND the 16-byte tensor-side stores are contiguous across neighbouring threads. In device_input_kernel those stores are Cp * 2
// bytes apart and fill sectors partially: at 64 channels it ran 3.3x slower than the NHWC input (H100 80GB HBM3, 400 W power limit,
// tools/device_io_bench.py).
// (The NCHW output reads such strided vectors, which cost it far less: it stays direct.) A tensor with a feed copy has <= 4 channels.
template <typename T>
__global__ void __launch_bounds__(256) device_input_nchw_tiled_kernel(const T* __restrict__ src, TV t, U8Norm q) {
    pdl_wait();
    __shared__ float s[64][33];
    const int HW = t.H * t.W, hw0 = blockIdx.x * 32, c0 = blockIdx.y * 64, n = blockIdx.z;
    const T* img = src + (size_t) n * t.C * HW;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int ch = ty + 8 * k, c = c0 + ch, hw = hw0 + tx;
        s[ch][tx] = (c < t.C && hw < HW) ? edge_in(img + (size_t) c * HW + hw, c, q) : 0.0f;
    }
    __syncthreads();
    const int g = threadIdx.x & 7, p = threadIdx.x >> 3; // 8 consecutive threads: the 8 channel groups of one pixel
    const int hw = hw0 + p, c = c0 + g * 8;
    if (hw >= HW || c >= t.Cp) return;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = s[g * 8 + j][p];
    store8(t.hi, t.lo, ((size_t) n * HW + hw) * t.Cp + c, v);
}
// A model output is never feed_only (MixedInferenceCore::init), so the regular planes are always the source.
template <typename T>
__global__ void device_output_kernel(TV t, T* __restrict__ dst, int nchw, float scale, float offset) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W * (t.Cp >> 3);
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const EdgeIndex e = edge_index(gid, t, nchw);
    float v[8];
    load8(t.hi, t.lo, e.px * t.Cp + e.c, v);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        if (e.c + j < t.C) edge_out(dst + e.base + (size_t) (e.c + j) * e.step, v[j], scale, offset);
}
int launch_device_input(snnb_context* ctx, const snnb_device_buffer& b, snnb_tensor* t) {
    U8Norm q;
    for (int i = 0; i < 4; ++i) q.mean[i] = b.mean4[i], q.norm[i] = b.norm4[i];
    const int nchw = b.layout == SNNB_LAYOUT_NCHW ? 1 : 0;
    if (nchw && t->c > 8 && !t->feed_hi) {
        const dim3 tiles((unsigned) ((t->h * t->w + 31) / 32), (unsigned) ((t->c + 63) / 64), (unsigned) t->n);
        switch (b.dtype) {
        case SNNB_DTYPE_F32:
            return launch_done(ctx, launch_k(device_input_nchw_tiled_kernel<float>, tiles, dim3(256), 0, ctx->stream, (const float*) b.data, view(t), q),
                               "device_input_nchw_tiled_kernel<f32>");
        case SNNB_DTYPE_F16:
            return launch_done(ctx, launch_k(device_input_nchw_tiled_kernel<__half>, tiles, dim3(256), 0, ctx->stream, (const __half*) b.data, view(t), q),
                               "device_input_nchw_tiled_kernel<f16>");
        case SNNB_DTYPE_U8:
            return launch_done(ctx, launch_k(device_input_nchw_tiled_kernel<uint8_t>, tiles, dim3(256), 0, ctx->stream, (const uint8_t*) b.data, view(t), q),
                               "device_input_nchw_tiled_kernel<u8>");
        }
    }
    const dim3 grid(vec_blocks(t, 256)), block(256);
    switch (b.dtype) {
    case SNNB_DTYPE_F32:
        return launch_done(ctx, launch_k(device_input_kernel<float>, grid, block, 0, ctx->stream, (const float*) b.data, nchw, view(t), q, feed_view(t)), "device_input_kernel<f32>");
    case SNNB_DTYPE_F16:
        return launch_done(ctx, launch_k(device_input_kernel<__half>, grid, block, 0, ctx->stream, (const __half*) b.data, nchw, view(t), q, feed_view(t)), "device_input_kernel<f16>");
    case SNNB_DTYPE_U8:
        return launch_done(ctx, launch_k(device_input_kernel<uint8_t>, grid, block, 0, ctx->stream, (const uint8_t*) b.data, nchw, view(t), q, feed_view(t)), "device_input_kernel<u8>");
    }
    SNNB_REQUIRE(false, "launch_device_input: unknown dtype %d", b.dtype);
}
int launch_device_output(snnb_context* ctx, const snnb_tensor* t, const snnb_device_buffer& b) {
    SNNB_REQUIRE(!t->feed_only, "launch_device_output: the tensor has no regular planes");
    const int nchw = b.layout == SNNB_LAYOUT_NCHW ? 1 : 0;
    const dim3 grid(vec_blocks(t, 256)), block(256);
    switch (b.dtype) {
    case SNNB_DTYPE_F32:
        return launch_done(ctx, launch_k(device_output_kernel<float>, grid, block, 0, ctx->stream, view(t), (float*) b.data, nchw, b.scale, b.offset), "device_output_kernel<f32>");
    case SNNB_DTYPE_F16:
        return launch_done(ctx, launch_k(device_output_kernel<__half>, grid, block, 0, ctx->stream, view(t), (__half*) b.data, nchw, b.scale, b.offset), "device_output_kernel<f16>");
    case SNNB_DTYPE_U8:
        return launch_done(ctx, launch_k(device_output_kernel<uint8_t>, grid, block, 0, ctx->stream, view(t), (uint8_t*) b.data, nchw, b.scale, b.offset), "device_output_kernel<u8>");
    }
    SNNB_REQUIRE(false, "launch_device_output: unknown dtype %d", b.dtype);
}

// Device video frames (snnb_model_run_frames) -> the model input: ImageTexture::resize's taps (resize_taps), each tap converted to
// RGBA8 with libyuv's integer YuvPixel (row_common.cc:1444-1484, the portable C rows), then resize_u8_kernel's blend, normalisation and
// stores. The constants are libyuv's YuvConstants written for U and V in their own roles; libyuv's NV12ToABGR reaches the same sums
// through the swapped kYvu* tables.
struct FrameV {
    const uint8_t* plane[3];
    int pitch[3];
    long long stride[3];
    int w, h;
    int yg, ub, ug, vg, vr, bb, bg, br;
};
// Not a public format: the Y plane (plane 0) of NV12 / NV21 / I420 frames as a 1-channel 8-bit image (snnb_model_transform_luma). Every
// component of its texel is the Y byte, so the model input is resize_u8_kernel's / split_u8_kernel's of that image.
constexpr int FRAME_LUMA = -1;
// Not a public format either: the Y plane of P010 frames, every component Y10 * 0.25 (the 10-bit sample in 8-bit units).
constexpr int FRAME_LUMA10 = -2;
// The 10-bit formats: their texels are exact multiples of 0.25 and are blended with blend_rn (restatable bit for bit in float32)
__host__ __device__ constexpr bool frame_10bit(int fmt) { return fmt == SNNB_FRAME_P010 || fmt == FRAME_LUMA10; }
// The 10-bit value of the 16-bit little-endian P010 sample at byte address p: the word's top 10 bits (P016's low 6 bits are ignored)
__device__ __forceinline__ int p010_sample(const uint8_t* p) { return __ldg(reinterpret_cast<const uint16_t*>(p)) >> 6; }
// RGBA8 of source pixel (x, y) of image n; pixel (x, y) takes chroma sample (x / 2, y / 2) (NV12ToARGBRow_C, row_common.cc:1945-1967).
// P010: libyuv's YuvPixel16 (Y with 10 bits, U and V truncated to 8) and StoreAR30's Clamp10(c >> 4), as R10 * 0.25, alpha 255.
template <int FMT>
__device__ __forceinline__ void frame_texel(const FrameV& s, int n, int x, int y, float rgba[4]) {
    if (FMT == FRAME_LUMA) {
        rgba[0] = rgba[1] = rgba[2] = rgba[3] = (float) __ldg(s.plane[0] + n * s.stride[0] + (size_t) y * s.pitch[0] + x);
        return;
    }
    if (FMT == FRAME_LUMA10) {
        rgba[0] = rgba[1] = rgba[2] = rgba[3] = (float) p010_sample(s.plane[0] + n * s.stride[0] + (size_t) y * s.pitch[0] + (size_t) x * 2) * 0.25f;
        return;
    }
    if (FMT == SNNB_FRAME_P010) {
        const int Y      = p010_sample(s.plane[0] + n * s.stride[0] + (size_t) y * s.pitch[0] + (size_t) x * 2);
        const uint8_t* c = s.plane[1] + n * s.stride[1] + (size_t) (y >> 1) * s.pitch[1] + (size_t) (x >> 1) * 4;
        const int U = p010_sample(c) >> 2, V = p010_sample(c + 2) >> 2;
        const int y1 = (int) ((uint32_t) ((Y << 6) * s.yg) >> 16);
        rgba[0] = (float) min(max((-(V * s.vr) + y1 + s.br) >> 4, 0), 1023) * 0.25f;
        rgba[1] = (float) min(max((-(U * s.ug + V * s.vg) + y1 + s.bg) >> 4, 0), 1023) * 0.25f;
        rgba[2] = (float) min(max((-(U * s.ub) + y1 + s.bb) >> 4, 0), 1023) * 0.25f;
        rgba[3] = 255.0f;
        return;
    }
    if (FMT == SNNB_FRAME_RGBA8) {
        const uint8_t* p = s.plane[0] + n * s.stride[0] + (size_t) y * s.pitch[0] + (size_t) x * 4;
#pragma unroll
        for (int c = 0; c < 4; ++c) rgba[c] = (float) __ldg(p + c);
        return;
    }
    const int Y = __ldg(s.plane[0] + n * s.stride[0] + (size_t) y * s.pitch[0] + x);
    int U, V;
    if (FMT == SNNB_FRAME_I420) {
        U = __ldg(s.plane[1] + n * s.stride[1] + (size_t) (y >> 1) * s.pitch[1] + (x >> 1));
        V = __ldg(s.plane[2] + n * s.stride[2] + (size_t) (y >> 1) * s.pitch[2] + (x >> 1));
    } else {
        const uint8_t* uv = s.plane[1] + n * s.stride[1] + (size_t) (y >> 1) * s.pitch[1] + (size_t) (x >> 1) * 2;
        U = __ldg(uv + (FMT == SNNB_FRAME_NV21 ? 1 : 0));
        V = __ldg(uv + (FMT == SNNB_FRAME_NV21 ? 0 : 1));
    }
    const int y1 = (int) ((uint32_t) (Y * 0x0101 * s.yg) >> 16);
    rgba[0] = (float) min(max((-(V * s.vr) + y1 + s.br) >> 6, 0), 255);
    rgba[1] = (float) min(max((-(U * s.ug + V * s.vg) + y1 + s.bg) >> 6, 0), 255);
    rgba[2] = (float) min(max((-(U * s.ub) + y1 + s.bb) >> 6, 0), 255);
    rgba[3] = 255.0f;
}
// The model input of one pixel (C <= 4: one 8-channel group) from its taps `r` in image n of the frames: each tap as libyuv's RGBA8,
// then resize_u8_kernel's blend (linear, unless the source is sampled directly) and normalisation. Shared by frame_input_kernel and
// frame_roi_input_kernel. The 10-bit formats blend with blend_rn instead, so that their model input is restatable in float32.
template <int FMT>
__device__ __forceinline__ void frame_pixel(const FrameV& s, int n, const ResizeTaps& r, int linear, bool direct, const TV& t, const U8Norm& q, float v[8]) {
    float p00[4];
    frame_texel<FMT>(s, n, r.x0, r.y0, p00);
    if (linear && !direct) {
        float p01[4], p10[4], p11[4];
        frame_texel<FMT>(s, n, r.x1, r.y0, p01);
        frame_texel<FMT>(s, n, r.x0, r.y1, p10);
        frame_texel<FMT>(s, n, r.x1, r.y1, p11);
        if constexpr (frame_10bit(FMT)) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                v[j] = (j < t.C) ? __fmul_rn(__fsub_rn(blend_rn(r, p00[j & 3], p01[j & 3], p10[j & 3], p11[j & 3]), q.mean[j & 3]), q.norm[j & 3]) : 0.0f;
            return;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (j < t.C) ? (r.blend(p00[j & 3], p01[j & 3], p10[j & 3], p11[j & 3]) - q.mean[j & 3]) * q.norm[j & 3] : 0.0f;
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (j < t.C) ? (p00[j & 3] - q.mean[j & 3]) * q.norm[j & 3] : 0.0f;
    }
}
// The stores of model-input pixel px: the regular planes (unless feed_only) and the stem feed copy
__device__ __forceinline__ void store_input_pixel(const TV& t, const FeedV& f, size_t px, const float v[8]) {
    if (!f.only) store8(t.hi, t.lo, px * 8, v);
    if (f.hi) store_feed(f, px, t.H, t.W, v);
}
// Where batch slot n's image comes from. Each kernel takes its source as a __grid_constant__ parameter: a reference to a kernel
// parameter that is not __grid_constant__ makes the compiler copy the parameter to local memory. frame_of(src, n) is the FrameV of image
// n, image_of(src, n) the image's index in it, and frame_size(src, f) the size of frame f. `form` names the source in launch errors.
// The batch's one FrameV is handed out by value: a reference to it made the YUV batch kernels 1.5-3.5 % slower (H100 SXM, 700 W).
// snnb_frames (snnb_model_run_frames): one description, image n at its image strides
struct FrameBatchV {
    FrameV s;
    static constexpr const char* form = "batch";
};
// Frame lists (snnb_model_run_frame_list): one FrameV per image, filled by frame_view, passed by value (26.6 KB at
// SNNB_FRAME_LIST_MAX images; CUDA 12.1+ allows 32,764 bytes). No allocation, no host-to-device copy, nothing that must outlive the
// launch, and a launch that a CUDA graph may capture. Indexed by a register, an entry is read from the constant bank (LDC).
struct FrameListV {
    FrameV img[SNNB_FRAME_LIST_MAX];
    static constexpr const char* form = "list";
};
__device__ __forceinline__ FrameV frame_of(const FrameBatchV& b, int) { return b.s; }
__device__ __forceinline__ int image_of(const FrameBatchV&, int n) { return n; }
__device__ __forceinline__ int2 frame_size(const FrameBatchV& b, int) { return make_int2(b.s.w, b.s.h); }
__device__ __forceinline__ const FrameV& frame_of(const FrameListV& L, int n) { return L.img[n]; }
__device__ __forceinline__ int image_of(const FrameListV&, int) { return 0; }
__device__ __forceinline__ int2 frame_size(const FrameListV& L, int f) { return make_int2(L.img[f].w, L.img[f].h); }

// Frame sizes alone, for roi_clear_kernel and the detection rows: every frame w x h (any number of frames), or frame n's own size from
// a table passed by value as FrameListV is (2 KB)
struct FrameSizeV {
    int w, h;
    static constexpr const char* form = "batch";
};
struct FrameSizesV {
    int wh[SNNB_FRAME_LIST_MAX][2];
    static constexpr const char* form = "list";
};
__device__ __forceinline__ int2 frame_size(const FrameSizeV& S, int) { return make_int2(S.w, S.h); }
__device__ __forceinline__ int2 frame_size(const FrameSizesV& S, int n) { return make_int2(S.wh[n][0], S.wh[n][1]); }
// One thread per output pixel (C <= 4: one 8-channel group). A frame of the model's size is sampled directly, as submitImpl does.
template <int FMT, class Src>
__global__ void __launch_bounds__(256) frame_input_kernel(const __grid_constant__ Src src, TV t, U8Norm q, int linear, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W;
    const size_t px    = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= total) return;
    const int ox = (int) (px % t.W), oy = (int) ((px / t.W) % t.H), n = (int) (px / ((size_t) t.W * t.H));
    const FrameV& s   = frame_of(src, n);
    const bool direct = s.w == t.W && s.h == t.H;
    ResizeTaps r;
    if (direct) r.x0 = r.x1 = ox, r.y0 = r.y1 = oy, r.ax = r.ay = 0.0f;
    else r = resize_taps(resize_pos(ox, oy, t.W, t.H, s.w, s.h), s.w, s.h, linear);
    float v[8];
    frame_pixel<FMT>(s, image_of(src, n), r, linear, direct, t, q, v);
    store_input_pixel(t, f, px, v);
}
// The kernel-side view of an snnb_frames: planes, size and libyuv's constants of its matrix
static FrameV frame_view(const snnb_frames& fr) {
    // libyuv row_common.cc:1115-1420: YG, YGB, UB, UG, VG, VR of BT.601 (kYuvI601Constants), BT.709 (kYuvH709Constants), BT.2020
    // (kYuv2020Constants) and full-range BT.601 (kYuvJPEGConstants). The biases UB * 128 + YGB etc. are libyuv's for all four.
    static const int M[4][6] = {
        {18997, -1160, -128, 25, 52, -102}, {18997, -1160, -128, 14, 34, -115}, {19003, -1160, -128, 12, 42, -107}, {16320, 32, -113, 22, 46, -90}};
    const int* m = M[fr.matrix == SNNB_YUV_BT709 ? 1 : (fr.matrix == SNNB_YUV_BT2020 ? 2 : (fr.matrix == (SNNB_YUV_BT601 | SNNB_YUV_FULL_RANGE) ? 3 : 0))];
    FrameV s;
    for (int i = 0; i < 3; ++i) s.plane[i] = fr.plane[i], s.pitch[i] = fr.pitch[i], s.stride[i] = fr.image_stride[i];
    s.w = fr.width, s.h = fr.height;
    s.yg = m[0], s.ub = m[2], s.ug = m[3], s.vg = m[4], s.vr = m[5];
    s.bb = m[2] * 128 + m[1], s.bg = m[3] * 128 + m[4] * 128 + m[1], s.br = m[5] * 128 + m[1];
    return s;
}
// The table of a list (checked by the caller: 1 <= count <= SNNB_FRAME_LIST_MAX); each entry is frame_view of the image as a one-image
// snnb_frames, so the matrix constants come from the same code. Entries past the count stay zero and are never read.
static void frame_list_view(const snnb_frame_list& fl, FrameListV& L) {
    std::memset(&L, 0, sizeof(L));
    for (int i = 0; i < fl.count; ++i) {
        const snnb_frame_image& im = fl.images[i];
        snnb_frames fr {};
        fr.format = fl.format, fr.matrix = im.matrix, fr.width = im.width, fr.height = im.height;
        for (int p = 0; p < 3; ++p) fr.plane[p] = im.plane[p], fr.pitch[p] = im.pitch[p];
        L.img[i] = frame_view(fr);
    }
}
static U8Norm frame_norm(const float mean4[4], const float norm4[4]) {
    U8Norm q;
    for (int i = 0; i < 4; ++i) q.mean[i] = mean4[i], q.norm[i] = norm4[i];
    return q;
}

// The kernel formats of a launch: every public format, the YUV ones (luma output), or the Y plane of YUV frames (FRAME_LUMA, and
// FRAME_LUMA10 for P010)
enum class FrameKernels { all, yuv, luma };
// Calls launch(std::integral_constant<int, FMT>()) with FMT the kernel format of `format` and returns its result; -1 when SET has no
// kernel for the format
template <FrameKernels SET, class F>
static int with_format(int format, F&& launch) {
    using std::integral_constant;
    if constexpr (SET == FrameKernels::luma) {
        if (format == SNNB_FRAME_P010) return launch(integral_constant<int, FRAME_LUMA10>());
        return launch(integral_constant<int, FRAME_LUMA>());
    } else {
        switch (format) {
        case SNNB_FRAME_NV12: return launch(integral_constant<int, SNNB_FRAME_NV12>());
        case SNNB_FRAME_NV21: return launch(integral_constant<int, SNNB_FRAME_NV21>());
        case SNNB_FRAME_I420: return launch(integral_constant<int, SNNB_FRAME_I420>());
        case SNNB_FRAME_P010: return launch(integral_constant<int, SNNB_FRAME_P010>());
        case SNNB_FRAME_RGBA8:
            if constexpr (SET == FrameKernels::all) return launch(integral_constant<int, SNNB_FRAME_RGBA8>());
            break;
        }
        return -1;
    }
}
static const char* format_name(int fmt) {
    switch (fmt) {
    case SNNB_FRAME_NV12: return "nv12";
    case SNNB_FRAME_NV21: return "nv21";
    case SNNB_FRAME_I420: return "i420";
    case SNNB_FRAME_RGBA8: return "rgba8";
    case SNNB_FRAME_P010: return "p010";
    case FRAME_LUMA: return "luma";
    case FRAME_LUMA10: return "luma10";
    }
    return "?";
}
// launch_done with the kernel named with its template arguments, kernel<arg0> or kernel<arg0, arg1>
static int launch_done(snnb_context* ctx, cudaError_t launched, const char* kernel, const char* arg0, const char* arg1 = nullptr) {
    char name[96];
    if (arg1) std::snprintf(name, sizeof(name), "%s<%s, %s>", kernel, arg0, arg1);
    else std::snprintf(name, sizeof(name), "%s<%s>", kernel, arg0);
    return launch_done(ctx, launched, name);
}

template <class Src>
static int frame_input(snnb_context* ctx, const char* who, const Src& src, int format, const U8Norm& q, int linear_filter, snnb_tensor* t, bool luma) {
    SNNB_REQUIRE(t->c <= 4 && t->cp == 8, "%s: the input tensor has %d channels; frames feed 1 to 4", who, t->c);
    if (luma)
        SNNB_REQUIRE(t->c == 1 && format != SNNB_FRAME_RGBA8, "%s: luma input feeds 1 channel from YUV frames (%d channels, format %d)", who, t->c, format);
    const int linear = linear_filter ? 1 : 0;
    const dim3 grid((unsigned) ((t->pixels() + 255) / 256)), block(256);
    auto launch = [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(frame_input_kernel<FMT, Src>, grid, block, 0, ctx->stream, src, view(t), q, linear, feed_view(t)), "frame_input_kernel",
                           format_name(FMT), Src::form);
    };
    const int rc = luma ? with_format<FrameKernels::luma>(format, launch) : with_format<FrameKernels::all>(format, launch);
    SNNB_REQUIRE(rc >= 0, "%s: unknown format %d", who, format);
    return rc;
}
int launch_frame_input(snnb_context* ctx, const snnb_frames& fr, snnb_tensor* t, bool luma) {
    return frame_input(ctx, "launch_frame_input", FrameBatchV {frame_view(fr)}, fr.format, frame_norm(fr.mean4, fr.norm4), fr.linear_filter, t, luma);
}
int launch_frame_input(snnb_context* ctx, const snnb_frame_list& fl, snnb_tensor* t, bool luma) {
    SNNB_REQUIRE(fl.count == t->n && fl.count <= SNNB_FRAME_LIST_MAX, "launch_frame_list_input: %d images for a batch of %d", fl.count, t->n);
    FrameListV L;
    frame_list_view(fl, L);
    return frame_input(ctx, "launch_frame_list_input", L, fl.format, frame_norm(fl.mean4, fl.norm4), fl.linear_filter, t, luma);
}

// Regions of device frames (snnb_model_run_rois / run_rois_list): batch slot n is region rois[n] of frame rois[n].frame. A used slot
// (n < the count) is valid when its region lies inside a frame that exists; roi_slot is the one test of that, so the input kernel and the
// clear kernel cannot disagree on which slots they serve.
struct RoiV {
    const snnb_roi* rois; // [N]
    const int* count;     // nullptr: every slot is used
    int num_frames;
};
// A frame index outside the frames fails the test, so the size looked up for it (of the nearest frame) does not matter
template <class Src>
__device__ __forceinline__ bool roi_slot(const Src& src, const RoiV& g, int slot, int N, snnb_roi& r) {
    const int* p = reinterpret_cast<const int*>(g.rois + slot);
    r.frame = __ldg(p), r.row = __ldg(p + 1), r.x = __ldg(p + 2), r.y = __ldg(p + 3), r.width = __ldg(p + 4), r.height = __ldg(p + 5);
    const int used = g.count ? min(max(__ldg(g.count), 0), N) : N;
    const int2 wh  = frame_size(src, min(max(r.frame, 0), g.num_frames - 1));
    return slot < used && r.frame >= 0 && r.frame < g.num_frames && r.width >= 1 && r.height >= 1 && r.x >= 0 && r.y >= 0 && r.x <= wh.x - r.width &&
           r.y <= wh.y - r.height;
}
// One thread per model-input pixel, as frame_input_kernel: the taps of ImageTexture::resize from a region-sized source, clamped to the
// region, then offset to the region's origin in the frame (so chroma is sited in frame coordinates). A region of the model's size is
// sampled directly. Invalid and unused slots get an all-zero input.
template <int FMT, class Src>
__global__ void __launch_bounds__(256) frame_roi_input_kernel(const __grid_constant__ Src src, RoiV g, TV t, U8Norm q, int linear, FeedV f) {
    pdl_wait();
    const size_t total = (size_t) t.N * t.H * t.W;
    const size_t px    = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (px >= total) return;
    const int ox = (int) (px % t.W), oy = (int) ((px / t.W) % t.H), n = (int) (px / ((size_t) t.W * t.H));
    snnb_roi roi;
    float v[8];
    if (roi_slot(src, g, n, t.N, roi)) {
        const bool direct = roi.width == t.W && roi.height == t.H;
        ResizeTaps r;
        if (direct) r.x0 = r.x1 = ox, r.y0 = r.y1 = oy, r.ax = r.ay = 0.0f;
        else r = resize_taps(resize_pos(ox, oy, t.W, t.H, roi.width, roi.height), roi.width, roi.height, linear);
        r.x0 += roi.x, r.x1 += roi.x, r.y0 += roi.y, r.y1 += roi.y;
        frame_pixel<FMT>(frame_of(src, roi.frame), image_of(src, roi.frame), r, linear, direct, t, q, v);
    } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.0f;
    }
    store_input_pixel(t, f, px, v);
}
template <class Src>
static int frame_roi_input(snnb_context* ctx, const char* who, const Src& src, int format, const U8Norm& q, int linear_filter, const RoiV& g, snnb_tensor* t) {
    SNNB_REQUIRE(t->c <= 4 && t->cp == 8, "%s: the input tensor has %d channels; frames feed 1 to 4", who, t->c);
    const int linear = linear_filter ? 1 : 0;
    const dim3 grid((unsigned) ((t->pixels() + 255) / 256)), block(256);
    const int rc = with_format<FrameKernels::all>(format, [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(frame_roi_input_kernel<FMT, Src>, grid, block, 0, ctx->stream, src, g, view(t), q, linear, feed_view(t)),
                           "frame_roi_input_kernel", format_name(FMT), Src::form);
    });
    SNNB_REQUIRE(rc >= 0, "%s: unknown format %d", who, format);
    return rc;
}
int launch_frame_roi_input(snnb_context* ctx, const snnb_frames& fr, int num_frames, const snnb_roi* rois, const int* count, snnb_tensor* t) {
    return frame_roi_input(ctx, "launch_frame_roi_input", FrameBatchV {frame_view(fr)}, fr.format, frame_norm(fr.mean4, fr.norm4), fr.linear_filter,
                           RoiV {rois, count, num_frames}, t);
}
int launch_frame_roi_input(snnb_context* ctx, const snnb_frame_list& fl, int num_frames, const snnb_roi* rois, const int* count, snnb_tensor* t) {
    SNNB_REQUIRE(num_frames == fl.count && fl.count >= 1 && fl.count <= SNNB_FRAME_LIST_MAX, "launch_frame_list_roi_input: %d frames", fl.count);
    FrameListV L;
    frame_list_view(fl, L);
    return frame_roi_input(ctx, "launch_frame_list_roi_input", L, fl.format, frame_norm(fl.mean4, fl.norm4), fl.linear_filter, RoiV {rois, count, fl.count}, t);
}
// Zeroes batch slot blockIdx.y of a caller's buffer (slot_bytes per slot, slots contiguous) when roi_slot rejects it. A slot is the
// outermost dimension in NHWC and NCHW alike. Runs after the outputs and classes are written.
template <class Src>
__global__ void __launch_bounds__(256) roi_clear_kernel(const __grid_constant__ Src src, RoiV g, int N, uint8_t* __restrict__ dst, long long slot_bytes) {
    pdl_wait();
    snnb_roi roi;
    if (roi_slot(src, g, (int) blockIdx.y, N, roi)) return;
    uint8_t* p = dst + (long long) blockIdx.y * slot_bytes;
    for (long long i = ((long long) blockIdx.x * blockDim.x + threadIdx.x) * 16; i < slot_bytes; i += (long long) gridDim.x * blockDim.x * 16) {
        if ((reinterpret_cast<uintptr_t>(p + i) & 15) == 0 && i + 16 <= slot_bytes) {
            *reinterpret_cast<uint4*>(p + i) = make_uint4(0u, 0u, 0u, 0u);
        } else {
            for (long long k = i; k < i + 16 && k < slot_bytes; ++k) p[k] = 0;
        }
    }
}
template <class Src>
static int roi_clear(snnb_context* ctx, const char* who, const Src& src, const RoiV& g, int batch, void* dst, long long slot_bytes) {
    SNNB_REQUIRE(batch >= 1 && batch <= 65535 && slot_bytes >= 1, "%s: batch %d, %lld bytes per slot", who, batch, slot_bytes);
    const long long chunks = (slot_bytes + 16 * 256 - 1) / (16 * 256);
    const dim3 grid((unsigned) std::min(chunks, 1024LL), (unsigned) batch);
    return launch_done(ctx, launch_k(roi_clear_kernel<Src>, grid, dim3(256), 0, ctx->stream, src, g, batch, static_cast<uint8_t*>(dst), slot_bytes),
                       "roi_clear_kernel", Src::form);
}
int launch_roi_clear(snnb_context* ctx, const snnb_frames& fr, int num_frames, const snnb_roi* rois, const int* count, int batch, void* dst, long long slot_bytes) {
    return roi_clear(ctx, "launch_roi_clear", FrameSizeV {fr.width, fr.height}, RoiV {rois, count, num_frames}, batch, dst, slot_bytes);
}
int launch_roi_clear(snnb_context* ctx, const snnb_frame_list& fl, int num_frames, const snnb_roi* rois, const int* count, int batch, void* dst,
                     long long slot_bytes) {
    SNNB_REQUIRE(num_frames == fl.count && fl.count >= 1 && fl.count <= SNNB_FRAME_LIST_MAX, "launch_roi_list_clear: %d frames", fl.count);
    FrameListV L;
    frame_list_view(fl, L);
    return roi_clear(ctx, "launch_roi_list_clear", L, RoiV {rois, count, fl.count}, batch, dst, slot_bytes);
}

// Detection rows -> regions (snnb_rois_from_detections). The rectangle of one row, every operation IEEE-rounded on its own (no FMA
// contraction), so that a float32 restatement reproduces it; false when the row is not kept.
__device__ __forceinline__ bool roi_from_row(const float* __restrict__ row, float W, float H, const snnb_roi_select& sel, snnb_roi& r) {
    const float cls = __ldg(row), score = __ldg(row + 1), x = __ldg(row + 2), y = __ldg(row + 3), w = __ldg(row + 4), h = __ldg(row + 5);
    if (!(score >= sel.min_score) || (sel.class_id != -1 && cls != (float) sel.class_id)) return false;
    const float ex = __fmul_rn(sel.expand, w), ey = __fmul_rn(sel.expand, h);
    const float fx0 = __fmul_rn(__fsub_rn(x, ex), W), fx1 = __fmul_rn(__fadd_rn(__fadd_rn(x, w), ex), W);
    const float fy0 = __fmul_rn(__fsub_rn(y, ey), H), fy1 = __fmul_rn(__fadd_rn(__fadd_rn(y, h), ey), H);
    if (isnan(fx0) || isnan(fx1) || isnan(fy0) || isnan(fy1)) return false;
    const int x0 = (int) floorf(fminf(fmaxf(fx0, 0.0f), W)), x1 = (int) ceilf(fminf(fmaxf(fx1, 0.0f), W));
    const int y0 = (int) floorf(fminf(fmaxf(fy0, 0.0f), H)), y1 = (int) ceilf(fminf(fmaxf(fy1, 0.0f), H));
    if (x1 <= x0 || y1 <= y0) return false;
    r.x = x0, r.y = y0, r.width = x1 - x0, r.height = y1 - y0;
    return true;
}
// One CTA visits rows (n, k), k < min(counts[n], max_rows), in order (frame, then row), a chunk of ROI_THREADS at a time: keep flags,
// a block prefix sum over them, and the kept rows scattered to their rank while it is below `capacity`. Then the tail is zeroed.
constexpr int ROI_THREADS = 1024;
template <class Sizes>
__global__ void __launch_bounds__(ROI_THREADS) rois_from_detections_kernel(const float* __restrict__ rows, const int* __restrict__ counts, int num_frames,
                                                                         int max_rows, const __grid_constant__ Sizes S, snnb_roi_select sel,
                                                                         snnb_roi* __restrict__ out, int capacity, int* __restrict__ count_out) {
    pdl_wait();
    __shared__ int warp_incl[ROI_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = ROI_THREADS / 32;
    const int total = num_frames * max_rows;
    int kept = 0; // rows kept before the current chunk (uniform over the CTA)
    for (int c0 = 0; c0 < total; c0 += ROI_THREADS) {
        const int i = c0 + threadIdx.x;
        snnb_roi r;
        bool keep = false;
        if (i < total) {
            const int n = i / max_rows, k = i - n * max_rows;
            if (k < min(__ldg(counts + n), max_rows)) {
                const int2 wh = frame_size(S, n);
                keep          = roi_from_row(rows + (size_t) i * 6, (float) wh.x, (float) wh.y, sel, r);
            }
            r.frame = n, r.row = k;
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) warp_incl[warp] = __popc(ballot);
        __syncthreads();
        if (warp == 0) {
            int v = warp_incl[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, v, d);
                if (lane >= d) v += u;
            }
            warp_incl[lane] = v;
        }
        __syncthreads();
        const int rank = kept + (warp ? warp_incl[warp - 1] : 0) + __popc(ballot & ((1u << lane) - 1u));
        if (keep && rank < capacity) out[rank] = r;
        kept += warp_incl[warps - 1];
        __syncthreads(); // warp_incl is rewritten by the next chunk
    }
    const int written = min(kept, capacity);
    for (int i = written + threadIdx.x; i < capacity; i += ROI_THREADS) out[i] = snnb_roi {0, 0, 0, 0, 0, 0};
    if (threadIdx.x == 0) *count_out = written;
}
template <class Sizes>
static int rois_from_detections_launch(snnb_context* ctx, cudaStream_t stream, const float* rows, const int* counts, int num_frames, int max_rows, const Sizes& S,
                                       const snnb_roi_select& sel, snnb_roi* rois, int capacity, int* count) {
    return launch_done(ctx, launch_k(rois_from_detections_kernel<Sizes>, dim3(1), dim3(ROI_THREADS), 0, stream, rows, counts, num_frames, max_rows, S, sel, rois,
                                     capacity, count),
                       "rois_from_detections_kernel", Sizes::form);
}
int launch_rois_from_detections(snnb_context* ctx, cudaStream_t stream, const float* rows, const int* counts, int num_frames, int max_rows, int fw, int fh,
                                const snnb_roi_select& sel, snnb_roi* rois, int capacity, int* count) {
    return rois_from_detections_launch(ctx, stream, rows, counts, num_frames, max_rows, FrameSizeV {fw, fh}, sel, rois, capacity, count);
}
int launch_rois_from_detections(snnb_context* ctx, cudaStream_t stream, const float* rows, const int* counts, int num_frames, int max_rows,
                                const int* frame_wh, const snnb_roi_select& sel, snnb_roi* rois, int capacity, int* count) {
    SNNB_REQUIRE(num_frames >= 1 && num_frames <= SNNB_FRAME_LIST_MAX, "launch_rois_from_detections_list: %d frames", num_frames);
    FrameSizesV S {};
    for (int n = 0; n < num_frames; ++n) S.wh[n][0] = frame_wh[2 * n], S.wh[n][1] = frame_wh[2 * n + 1];
    return rois_from_detections_launch(ctx, stream, rows, counts, num_frames, max_rows, S, sel, rois, capacity, count);
}

// Detection on regions (snnb_model_detect_rois): the per-slot rows of launch_yolo_detect (max_rows 100) mapped to their frames and
// merged by one greedy NMS per frame. Frame f's segment is the mapped rows of every valid slot on f, slots in order and each slot's rows
// in order; the segments lie frame after frame in `seg`, so segment f starts after the rows of the valid slots on frames below f.
// Three kernels, none with atomics: roi_merge_gather_kernel (one CTA per frame) finds its segment and fills it, roi_merge_rank_kernel
// sorts each segment by rank as yolo_rank_kernel does, roi_merge_nms_kernel (one CTA per frame) runs yolo_greedy_nms over it.
constexpr int MERGE_THREADS = 256;
// Exclusive prefix sum of v over the CTA (MERGE_THREADS threads); total = the sum. sh: MERGE_THREADS / 32 ints of shared memory.
__device__ __forceinline__ int merge_scan(int v, int* sh, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += u;
    }
    if (lane == 31) sh[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = lane < MERGE_THREADS / 32 ? sh[lane] : 0;
#pragma unroll
        for (int d = 1; d < MERGE_THREADS / 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += u;
        }
        if (lane < MERGE_THREADS / 32) sh[lane] = w;
    }
    __syncthreads();
    const int excl = incl - v + (warp ? sh[warp - 1] : 0);
    total          = sh[MERGE_THREADS / 32 - 1];
    __syncthreads(); // sh is rewritten by the next scan
    return excl;
}
// Frame blockIdx.x: two walks over the N slots in order. The first sums the rows of the valid slots on lower frames (the segment's
// start), the second places each valid slot on this frame after the ones before it and writes its rows, mapped to the frame:
// {cls, score, (rx + x * rw) / W, (ry + y * rh) / H, (w * rw) / W, (h * rh) / H}, every operation rounded on its own.
// segs[f] = {start, length}.
template <class Sizes>
__global__ void __launch_bounds__(MERGE_THREADS) roi_merge_gather_kernel(const __grid_constant__ Sizes S, RoiV g, int N, const float* __restrict__ slot_rows,
                                                                        const int* __restrict__ slot_counts, YoloBox* __restrict__ seg,
                                                                        int2* __restrict__ segs) {
    using yolo_dev::MAX_ROWS;
    pdl_wait();
    __shared__ int sh[MERGE_THREADS / 32];
    __shared__ int off[MERGE_THREADS], cnt[MERGE_THREADS];
    __shared__ int4 reg[MERGE_THREADS];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int2 wh = frame_size(S, f);
    const float W = (float) wh.x, H = (float) wh.y;
    int start = 0, len = 0, total;
    for (int s0 = 0; s0 < N; s0 += MERGE_THREADS) {
        const int s = s0 + tid;
        snnb_roi roi;
        const int below = s < N && roi_slot(S, g, s, N, roi) && roi.frame < f ? __ldg(slot_counts + s) : 0;
        merge_scan(below, sh, total);
        start += total;
    }
    for (int s0 = 0; s0 < N; s0 += MERGE_THREADS) {
        const int s = s0 + tid;
        snnb_roi roi {0, 0, 0, 0, 0, 0};
        const int mine = s < N && roi_slot(S, g, s, N, roi) && roi.frame == f ? __ldg(slot_counts + s) : 0;
        off[tid] = start + len + merge_scan(mine, sh, total);
        cnt[tid] = mine;
        reg[tid] = make_int4(roi.x, roi.y, roi.width, roi.height);
        __syncthreads();
        const int rows = min(MERGE_THREADS, N - s0) * MAX_ROWS;
        for (int e = tid; e < rows; e += MERGE_THREADS) {
            const int j = e / MAX_ROWS, k = e - j * MAX_ROWS;
            if (k >= cnt[j]) continue;
            const float* row = slot_rows + ((size_t) (s0 + j) * MAX_ROWS + k) * 6;
            const int4 q   = reg[j];
            const float rx = (float) q.x, ry = (float) q.y, rw = (float) q.z, rh = (float) q.w;
            const float x = __ldg(row + 2), y = __ldg(row + 3), w = __ldg(row + 4), h = __ldg(row + 5);
            seg[off[j] + k] = YoloBox {(int) __ldg(row), __ldg(row + 1), __fdiv_rn(__fadd_rn(rx, __fmul_rn(x, rw)), W), __fdiv_rn(__fadd_rn(ry, __fmul_rn(y, rh)), H),
                                       __fdiv_rn(__fmul_rn(w, rw), W), __fdiv_rn(__fmul_rn(h, rh), H)};
        }
        len += total;
        __syncthreads(); // off, cnt and reg are rewritten by the next chunk
    }
    if (tid == 0) segs[f] = make_int2(start, len);
}
// Rank sort of segment blockIdx.x (yolo_rank_kernel's): std::stable_sort by descending score over the segment == descending
// (score, -position), yolo_key(score, position). Blocks past the segment's length exit at once.
__global__ void __launch_bounds__(MERGE_THREADS) roi_merge_rank_kernel(const int2* __restrict__ segs, const YoloBox* __restrict__ seg, YoloBox* __restrict__ sorted) {
    pdl_wait();
    __shared__ unsigned long long tile[MERGE_THREADS];
    const int2 sg = segs[blockIdx.x];
    const int count = sg.y;
    if ((int) (blockIdx.y * blockDim.x) >= count) return;
    const YoloBox* b = seg + sg.x;
    const int i      = blockIdx.y * blockDim.x + threadIdx.x;
    const unsigned long long mine = i < count ? yolo_key(b[i].score, i) : 0ull;
    int rank = 0;
    for (int t0 = 0; t0 < count; t0 += MERGE_THREADS) {
        __syncthreads();
        if (t0 + (int) threadIdx.x < count) tile[threadIdx.x] = yolo_key(b[t0 + threadIdx.x].score, t0 + threadIdx.x);
        __syncthreads();
        const int m = min(MERGE_THREADS, count - t0);
        for (int j = 0; j < m; ++j) rank += tile[j] > mine ? 1 : 0;
    }
    if (i < count) sorted[sg.x + rank] = b[i];
}
// A sorted segment's boxes, as decoded and mapped
struct MergedBoxes {
    const YoloBox* b;
    __device__ __forceinline__ bool operator()(int i, YoloBox& o) const {
        o = b[i];
        return true;
    }
};
// Greedy NMS of frame blockIdx.x's sorted segment: rows[f][max_rows][6], counts[f]
__global__ void __launch_bounds__(yolo_dev::NMS_THREADS) roi_merge_nms_kernel(const int2* __restrict__ segs, const YoloBox* __restrict__ sorted, int max_rows,
                                                                             float* __restrict__ rows, int* __restrict__ counts) {
    pdl_wait();
    const int f   = blockIdx.x;
    const int2 sg = segs[f];
    yolo_greedy_nms(MergedBoxes {sorted + sg.x}, sg.y, max_rows, f, rows, counts);
}
size_t roi_merge_scratch_bytes(int batch) { return (size_t) batch * yolo_dev::MAX_ROWS * 2 * sizeof(YoloBox); }
template <class Sizes>
static int roi_merge(snnb_context* ctx, const Sizes& S, const RoiV& g, int batch, const float* slot_rows, const int* slot_counts, void* scratch, int2* segs,
                     int max_rows, float* rows, int* counts) {
    SNNB_REQUIRE(batch >= 1 && batch <= 65535 && g.num_frames >= 1 && max_rows >= 1 && max_rows <= yolo_dev::MAX_ROWS,
                 "launch_roi_merge: batch %d, %d frames, max_rows %d", batch, g.num_frames, max_rows);
    auto* seg    = static_cast<YoloBox*>(scratch);
    auto* sorted = seg + (size_t) batch * yolo_dev::MAX_ROWS;
    const unsigned frames = (unsigned) g.num_frames;
    if (launch_done(ctx, launch_k(roi_merge_gather_kernel<Sizes>, dim3(frames), dim3(MERGE_THREADS), 0, ctx->stream, S, g, batch, slot_rows, slot_counts, seg, segs),
                    "roi_merge_gather_kernel", Sizes::form))
        return 1;
    const dim3 rank_grid(frames, (unsigned) ((batch * yolo_dev::MAX_ROWS + MERGE_THREADS - 1) / MERGE_THREADS));
    if (launch_done(ctx, launch_k(roi_merge_rank_kernel, rank_grid, dim3(MERGE_THREADS), 0, ctx->stream, (const int2*) segs, (const YoloBox*) seg, sorted),
                    "roi_merge_rank_kernel"))
        return 1;
    return launch_done(ctx, launch_k(roi_merge_nms_kernel, dim3(frames), dim3(yolo_dev::NMS_THREADS), 0, ctx->stream, (const int2*) segs, (const YoloBox*) sorted,
                                     max_rows, rows, counts),
                       "roi_merge_nms_kernel");
}
int launch_roi_merge(snnb_context* ctx, const snnb_frames& fr, int num_frames, const snnb_roi* rois, const int* count, int batch, const float* slot_rows,
                     const int* slot_counts, void* scratch, void* segs, int max_rows, float* rows, int* counts) {
    return roi_merge(ctx, FrameSizeV {fr.width, fr.height}, RoiV {rois, count, num_frames}, batch, slot_rows, slot_counts, scratch, static_cast<int2*>(segs), max_rows,
                     rows, counts);
}
int launch_roi_merge(snnb_context* ctx, const snnb_frame_list& fl, int num_frames, const snnb_roi* rois, const int* count, int batch, const float* slot_rows,
                     const int* slot_counts, void* scratch, void* segs, int max_rows, float* rows, int* counts) {
    SNNB_REQUIRE(num_frames == fl.count && fl.count >= 1 && fl.count <= SNNB_FRAME_LIST_MAX, "launch_roi_list_merge: %d frames", fl.count);
    FrameSizesV S {};
    for (int n = 0; n < fl.count; ++n) S.wh[n][0] = fl.images[n].width, S.wh[n][1] = fl.images[n].height;
    return roi_merge(ctx, S, RoiV {rois, count, fl.count}, batch, slot_rows, slot_counts, scratch, static_cast<int2*>(segs), max_rows, rows, counts);
}

// The selector node of a region call's dispatch graph (snnb_model_set_count_batches): turns on the one IF body whose size count_body
// picks for *count; the other handles keep their default of 0, and a count of 0 (or below) turns on none. The bodies' sizes are read
// from the __grid_constant__ parameter, so indexing them makes no local copy.
__global__ void __launch_bounds__(1) count_select_kernel(const int* __restrict__ count, const __grid_constant__ CountBodies b) {
    const int s = count_body(b.size, b.num - 1, b.size[b.num - 1], *count);
    for (int k = 0; k < b.num; ++k)
        if (b.size[k] == s) {
            cudaGraphSetConditional(b.handle[k], 1u);
            return;
        }
}
static cudaKernelNodeParams count_select_params(void** args) {
    cudaKernelNodeParams p = {};
    p.func         = reinterpret_cast<void*>(count_select_kernel);
    p.gridDim      = dim3(1);
    p.blockDim     = dim3(1);
    p.kernelParams = args;
    return p;
}
int count_select_add(cudaGraph_t g, cudaGraphNode_t* node, const int* count, const CountBodies& b) {
    void* args[] = {&count, const_cast<CountBodies*>(&b)};
    const cudaKernelNodeParams p = count_select_params(args);
    SNNB_CUDA_OK(cudaGraphAddKernelNode(node, g, nullptr, 0, &p));
    return 0;
}
int count_select_set(cudaGraphExec_t exec, cudaGraphNode_t node, const int* count, const CountBodies& b) {
    void* args[] = {&count, const_cast<CountBodies*>(&b)};
    const cudaKernelNodeParams p = count_select_params(args);
    SNNB_CUDA_OK(cudaGraphExecKernelNodeSetParams(exec, node, &p));
    return 0;
}

// Model output 0 -> device video frames (snnb_model_transform_frames), the reverse of frame_input_kernel. Each frame pixel is
// ImageTexture::resize (resize_taps) of M, the model-size RGBA8 image whose texels are quant_u8 of the output's channels; then libyuv's
// ABGRToNV12 / ABGRToNV21 / ABGRToI420 with its portable C rows (row_common.cc:423-473: RGBToY, RGBToU, RGBToV and MAKEROWY's 2 x 2
// chroma average).
struct FrameOutV {
    uint8_t* plane[3];
    int pitch[3];
    long long stride[3];
    int w, h;
    float scale, offset;
};
// A model output value as 10 bits (P010 output): clamp(rint(4 * (v * scale + offset)), 0, 1023), the product and the sum each rounded
// on its own, so that numpy float32 restates it exactly. The same scale and offset as for 8-bit output give the same range.
__device__ __forceinline__ float quant10(float v, float scale, float offset) {
    return fminf(fmaxf(rintf(4.0f * __fadd_rn(__fmul_rn(v, scale), offset)), 0.0f), 1023.0f);
}
template <bool TEN>
__device__ __forceinline__ float quant_out(float v, float scale, float offset) {
    if constexpr (TEN) return quant10(v, scale, offset);
    else return quant_u8(v, scale, offset);
}
// Texel (x, y) of image n of M: C = 4 RGBA, C = 3 RGB + alpha 255, C = 1 grey (R = G = B) + alpha 255. TEN: 10-bit components (M10).
template <bool TEN>
__device__ __forceinline__ void out_texel(const TV& t, int n, int x, int y, float scale, float offset, float rgba[4]) {
    float v[8];
    load8(t.hi, t.lo, (((size_t) n * t.H + y) * t.W + x) * t.Cp, v);
    if (t.C == 1) {
        rgba[0] = rgba[1] = rgba[2] = quant_out<TEN>(v[0], scale, offset);
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) rgba[c] = quant_out<TEN>(v[c], scale, offset);
    }
    rgba[3] = t.C == 4 ? quant_out<TEN>(v[3], scale, offset) : 255.0f;
}
// Pixel (x, y) of image n of the frame-size RGBA8 image F (TEN: its 10-bit counterpart from M10). A frame of the output's size takes M
// as it is.
template <bool TEN>
__device__ __forceinline__ void frame_out_pixel(const TV& t, const FrameOutV& o, int n, int x, int y, int linear, int rgba[4]) {
    const bool direct = o.w == t.W && o.h == t.H;
    ResizeTaps r;
    if (direct) r.x0 = r.x1 = x, r.y0 = r.y1 = y, r.ax = r.ay = 0.0f;
    else r = resize_taps(resize_pos(x, y, o.w, o.h, t.W, t.H), t.W, t.H, linear);
    float p00[4];
    out_texel<TEN>(t, n, r.x0, r.y0, o.scale, o.offset, p00);
    if (linear && !direct) {
        float p01[4], p10[4], p11[4];
        out_texel<TEN>(t, n, r.x1, r.y0, o.scale, o.offset, p01);
        out_texel<TEN>(t, n, r.x0, r.y1, o.scale, o.offset, p10);
        out_texel<TEN>(t, n, r.x1, r.y1, o.scale, o.offset, p11);
#pragma unroll
        for (int c = 0; c < 4; ++c) rgba[c] = (int) rintf(blend_rn(r, p00[c], p01[c], p10[c], p11[c]));
    } else {
#pragma unroll
        for (int c = 0; c < 4; ++c) rgba[c] = (int) p00[c];
    }
}
// Two bytes at p, in one store where p is 2-byte aligned
__device__ __forceinline__ void store_2u8(uint8_t* p, int a, int b) {
    if ((reinterpret_cast<uintptr_t>(p) & 1) == 0) *reinterpret_cast<uint16_t*>(p) = (uint16_t) (a | (b << 8));
    else p[0] = (uint8_t) a, p[1] = (uint8_t) b;
}
// Two 10-bit values at p as P010 words (value << 6, low 6 bits zero), in one store where p is 4-byte aligned (p is 2-byte aligned)
__device__ __forceinline__ void store_2p010(uint8_t* p, int a, int b) {
    if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) *reinterpret_cast<uint32_t*>(p) = (uint32_t) (a << 6) | ((uint32_t) (b << 6) << 16);
    else reinterpret_cast<uint16_t*>(p)[0] = (uint16_t) (a << 6), reinterpret_cast<uint16_t*>(p)[1] = (uint16_t) (b << 6);
}
// The 2 x 2 block (bx, by) of frame pixels of image n, i.e. one chroma sample: its 4 pixels of F, then 4 Y bytes and the chroma sample
// (or 4 RGBA8 pixels). Pixels past an odd width or height are not written. P010: the same from M10, with the 8-bit coefficients and the
// 10-bit offsets (64 and 512), stored as 16-bit words. Shared by frame_output_kernel and frame_list_output_kernel.
template <int FMT>
__device__ __forceinline__ void frame_out_block(const TV& t, const FrameOutV& o, int n, int bx, int by, int linear) {
    constexpr bool TEN = FMT == SNNB_FRAME_P010;
    const int x = 2 * bx, y = 2 * by;
    const bool has_x1 = x + 1 < o.w, has_y1 = y + 1 < o.h;
    int p[2][2][4];
    frame_out_pixel<TEN>(t, o, n, x, y, linear, p[0][0]);
    if (has_x1) frame_out_pixel<TEN>(t, o, n, x + 1, y, linear, p[0][1]);
    if (has_y1) frame_out_pixel<TEN>(t, o, n, x, y + 1, linear, p[1][0]);
    if (has_x1 && has_y1) frame_out_pixel<TEN>(t, o, n, x + 1, y + 1, linear, p[1][1]);
    if constexpr (TEN) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            if (dy && !has_y1) break;
            uint8_t* d = o.plane[0] + n * o.stride[0] + (size_t) (y + dy) * o.pitch[0] + (size_t) x * 2;
            const int* a = p[dy][0];
            const int ya = (66 * a[0] + 129 * a[1] + 25 * a[2] + 0x4080) >> 8;
            if (has_x1) {
                const int* b = p[dy][1];
                store_2p010(d, ya, (66 * b[0] + 129 * b[1] + 25 * b[2] + 0x4080) >> 8);
            } else {
                *reinterpret_cast<uint16_t*>(d) = (uint16_t) (ya << 6);
            }
        }
    }
    if (FMT == SNNB_FRAME_RGBA8) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                if ((dx && !has_x1) || (dy && !has_y1)) continue;
                const int* q = p[dy][dx];
                uint8_t* d = o.plane[0] + n * o.stride[0] + (size_t) (y + dy) * o.pitch[0] + (size_t) (x + dx) * 4;
                if ((reinterpret_cast<uintptr_t>(d) & 3) == 0) *reinterpret_cast<uint32_t*>(d) = (uint32_t) (q[0] | (q[1] << 8) | (q[2] << 16) | (q[3] << 24));
                else d[0] = (uint8_t) q[0], d[1] = (uint8_t) q[1], d[2] = (uint8_t) q[2], d[3] = (uint8_t) q[3];
            }
        return;
    }
    if constexpr (!TEN) {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
            if (dy && !has_y1) break;
            uint8_t* d = o.plane[0] + n * o.stride[0] + (size_t) (y + dy) * o.pitch[0] + x;
            const int* a = p[dy][0];
            const int ya = (66 * a[0] + 129 * a[1] + 25 * a[2] + 0x1080) >> 8;
            if (has_x1) {
                const int* b = p[dy][1];
                store_2u8(d, ya, (66 * b[0] + 129 * b[1] + 25 * b[2] + 0x1080) >> 8);
            } else {
                d[0] = (uint8_t) ya;
            }
        }
    }
    // libyuv pairs an odd last row with itself (ABGRToUVRow with stride 0) and averages an odd last column over its two rows
    int avg[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int a = p[0][0][c], cc = has_y1 ? p[1][0][c] : a;
        if (has_x1) {
            const int b = p[0][1][c], dd = has_y1 ? p[1][1][c] : b;
            avg[c] = (a + b + cc + dd) >> 2;
        } else {
            avg[c] = (a + cc) >> 1;
        }
    }
    constexpr int COFF = TEN ? 0x20080 : 0x8080;
    const int U = (112 * avg[2] - 74 * avg[1] - 38 * avg[0] + COFF) >> 8, V = (112 * avg[0] - 94 * avg[1] - 18 * avg[2] + COFF) >> 8;
    if (TEN) {
        store_2p010(o.plane[1] + n * o.stride[1] + (size_t) by * o.pitch[1] + (size_t) bx * 4, U, V);
    } else if (FMT == SNNB_FRAME_I420) {
        o.plane[1][n * o.stride[1] + (size_t) by * o.pitch[1] + bx] = (uint8_t) U;
        o.plane[2][n * o.stride[2] + (size_t) by * o.pitch[2] + bx] = (uint8_t) V;
    } else {
        uint8_t* d = o.plane[1] + n * o.stride[1] + (size_t) by * o.pitch[1] + (size_t) bx * 2;
        if (FMT == SNNB_FRAME_NV12) store_2u8(d, U, V);
        else store_2u8(d, V, U);
    }
}
// One thread per 2 x 2 block of frame pixels (frame_out_block)
template <int FMT>
__global__ void __launch_bounds__(256) frame_output_kernel(TV t, FrameOutV o, int linear) {
    pdl_wait();
    const int cw = (o.w + 1) >> 1, ch = (o.h + 1) >> 1;
    const size_t total = (size_t) t.N * ch * cw;
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int bx = (int) (gid % cw), by = (int) ((gid / cw) % ch), n = (int) (gid / ((size_t) cw * ch));
    frame_out_block<FMT>(t, o, n, bx, by, linear);
}
int launch_frame_output(snnb_context* ctx, const snnb_tensor* t, const snnb_frames_out& fr) {
    SNNB_REQUIRE((t->c == 1 || t->c == 3 || t->c == 4) && t->cp == 8 && !t->feed_only, "launch_frame_output: the output tensor has %d channels; frames are written from 1, 3 or 4",
                 t->c);
    FrameOutV o;
    for (int i = 0; i < 3; ++i) o.plane[i] = fr.plane[i], o.pitch[i] = fr.pitch[i], o.stride[i] = fr.image_stride[i];
    o.w = fr.width, o.h = fr.height, o.scale = fr.scale, o.offset = fr.offset;
    const int linear = fr.linear_filter ? 1 : 0;
    const size_t blocks = (size_t) t->n * ((fr.height + 1) / 2) * ((fr.width + 1) / 2);
    const dim3 grid((unsigned) ((blocks + 255) / 256)), block(256);
    const int rc = with_format<FrameKernels::all>(fr.format, [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(frame_output_kernel<FMT>, grid, block, 0, ctx->stream, view(t), o, linear), "frame_output_kernel", format_name(FMT));
    });
    SNNB_REQUIRE(rc >= 0, "launch_frame_output: unknown format %d", fr.format);
    return rc;
}

// A 1-channel model output 0 -> the Y plane of device video frames, with the source frames' chroma resampled beside it
// (snnb_model_transform_luma). Y is frame_out_pixel's component 0 from one value per texel; U and V are ImageTexture::resize of the
// source chroma planes, plane to plane, with the same taps and blend_rn.
// Texel (x, y) of image n of M (TEN: M10) for a 1-channel output: its one value, quantised
template <bool TEN>
__device__ __forceinline__ float out_luma_texel(const TV& t, int n, int x, int y, float scale, float offset) {
    const size_t off = (((size_t) n * t.H + y) * t.W + x) * t.Cp;
    const float v    = __half2float(__ldg(t.hi + off)) + (t.lo ? __half2float(__ldg(t.lo + off)) : 0.0f); // = load8's component 0
    return quant_out<TEN>(v, scale, offset);
}
template <bool TEN>
__device__ __forceinline__ int luma_out_pixel(const TV& t, const FrameOutV& o, int n, int x, int y, int linear) {
    const bool direct = o.w == t.W && o.h == t.H;
    ResizeTaps r;
    if (direct) r.x0 = r.x1 = x, r.y0 = r.y1 = y, r.ax = r.ay = 0.0f;
    else r = resize_taps(resize_pos(x, y, o.w, o.h, t.W, t.H), t.W, t.H, linear);
    const float p00 = out_luma_texel<TEN>(t, n, r.x0, r.y0, o.scale, o.offset);
    if (!linear || direct) return (int) p00;
    const float p01 = out_luma_texel<TEN>(t, n, r.x1, r.y0, o.scale, o.offset), p10 = out_luma_texel<TEN>(t, n, r.x0, r.y1, o.scale, o.offset);
    const float p11 = out_luma_texel<TEN>(t, n, r.x1, r.y1, o.scale, o.offset);
    return (int) rintf(blend_rn(r, p00, p01, p10, p11));
}
// Chroma sample (x, y) of image n: U from plane 1, V from plane 2 of `s`, `step` samples apart along a row (2 in an interleaved plane).
// TEN: 16-bit P010 samples, as their 10-bit values.
template <bool TEN>
__device__ __forceinline__ void chroma_texel(const FrameV& s, int step, int n, int x, int y, float& u, float& v) {
    if constexpr (TEN) {
        u = (float) p010_sample(s.plane[1] + n * s.stride[1] + (size_t) y * s.pitch[1] + (size_t) x * step * 2);
        v = (float) p010_sample(s.plane[2] + n * s.stride[2] + (size_t) y * s.pitch[2] + (size_t) x * step * 2);
    } else {
        u = (float) __ldg(s.plane[1] + n * s.stride[1] + (size_t) y * s.pitch[1] + (size_t) x * step);
        v = (float) __ldg(s.plane[2] + n * s.stride[2] + (size_t) y * s.pitch[2] + (size_t) x * step);
    }
}
// The 2 x 2 block (bx, by) of frame pixels of image n, i.e. one chroma sample: 4 Y bytes, then the chroma sample resized from the
// source's chroma planes. A chroma plane of the source's size is copied. Pixels past an odd width or height are not written. P010 (from
// P010 frames): 10-bit Y from M10 and the source's 10-bit chroma, each stored as value << 6. Shared by luma_output_kernel and
// luma_list_output_kernel.
template <int FMT>
__device__ __forceinline__ void luma_out_block(const TV& t, const FrameV& s, int step, const FrameOutV& o, int n, int bx, int by, int linear) {
    constexpr bool TEN = FMT == SNNB_FRAME_P010;
    const int cw = (o.w + 1) >> 1, ch = (o.h + 1) >> 1;
    const int x = 2 * bx, y = 2 * by;
    const bool has_x1 = x + 1 < o.w, has_y1 = y + 1 < o.h;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
        if (dy && !has_y1) break;
        if constexpr (TEN) {
            uint8_t* d   = o.plane[0] + n * o.stride[0] + (size_t) (y + dy) * o.pitch[0] + (size_t) x * 2;
            const int ya = luma_out_pixel<true>(t, o, n, x, y + dy, linear);
            if (has_x1) store_2p010(d, ya, luma_out_pixel<true>(t, o, n, x + 1, y + dy, linear));
            else *reinterpret_cast<uint16_t*>(d) = (uint16_t) (ya << 6);
        } else {
            uint8_t* d   = o.plane[0] + n * o.stride[0] + (size_t) (y + dy) * o.pitch[0] + x;
            const int ya = luma_out_pixel<false>(t, o, n, x, y + dy, linear);
            if (has_x1) store_2u8(d, ya, luma_out_pixel<false>(t, o, n, x + 1, y + dy, linear));
            else d[0] = (uint8_t) ya;
        }
    }
    const int scw = (s.w + 1) >> 1, sch = (s.h + 1) >> 1;
    const bool direct = cw == scw && ch == sch;
    ResizeTaps r;
    if (direct) r.x0 = r.x1 = bx, r.y0 = r.y1 = by, r.ax = r.ay = 0.0f;
    else r = resize_taps(resize_pos(bx, by, cw, ch, scw, sch), scw, sch, linear);
    float u00, v00;
    chroma_texel<TEN>(s, step, n, r.x0, r.y0, u00, v00);
    int U = (int) u00, V = (int) v00;
    if (linear && !direct) {
        float u01, v01, u10, v10, u11, v11;
        chroma_texel<TEN>(s, step, n, r.x1, r.y0, u01, v01);
        chroma_texel<TEN>(s, step, n, r.x0, r.y1, u10, v10);
        chroma_texel<TEN>(s, step, n, r.x1, r.y1, u11, v11);
        U = (int) rintf(blend_rn(r, u00, u01, u10, u11)), V = (int) rintf(blend_rn(r, v00, v01, v10, v11));
    }
    if (TEN) {
        store_2p010(o.plane[1] + n * o.stride[1] + (size_t) by * o.pitch[1] + (size_t) bx * 4, U, V);
    } else if (FMT == SNNB_FRAME_I420) {
        o.plane[1][n * o.stride[1] + (size_t) by * o.pitch[1] + bx] = (uint8_t) U;
        o.plane[2][n * o.stride[2] + (size_t) by * o.pitch[2] + bx] = (uint8_t) V;
    } else {
        uint8_t* d = o.plane[1] + n * o.stride[1] + (size_t) by * o.pitch[1] + (size_t) bx * 2;
        if (FMT == SNNB_FRAME_NV12) store_2u8(d, U, V);
        else store_2u8(d, V, U);
    }
}
// One thread per 2 x 2 block of frame pixels (luma_out_block), as frame_output_kernel
template <int FMT>
__global__ void __launch_bounds__(256) luma_output_kernel(TV t, FrameV s, int step, FrameOutV o, int linear) {
    pdl_wait();
    const int cw = (o.w + 1) >> 1, ch = (o.h + 1) >> 1;
    const size_t total = (size_t) t.N * ch * cw;
    const size_t gid   = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= total) return;
    const int bx = (int) (gid % cw), by = (int) ((gid / cw) % ch), n = (int) (gid / ((size_t) cw * ch));
    luma_out_block<FMT>(t, s, step, o, n, bx, by, linear);
}
// Where luma_out_block reads the source chroma of `format` frames: U and V from planes plane[0] and plane[1] at byte offsets offset[0] and
// offset[1], `step` samples apart along a row. I420: planes 1 and 2; NV12 / NV21 / P010: the two samples of each pair in plane 1.
struct ChromaSource {
    int plane[2], offset[2], step;
};
static ChromaSource chroma_source(int format) {
    if (format == SNNB_FRAME_I420) return {{1, 2}, {0, 0}, 1};
    const int u = format == SNNB_FRAME_NV21 ? 1 : 0, bytes = format == SNNB_FRAME_P010 ? 2 : 1;
    return {{1, 1}, {u * bytes, (1 - u) * bytes}, 2};
}
int launch_luma_output(snnb_context* ctx, const snnb_tensor* t, const snnb_frames& src, const snnb_frames_out& fr) {
    SNNB_REQUIRE(t->c == 1 && t->cp == 8 && !t->feed_only && src.format != SNNB_FRAME_RGBA8,
                 "launch_luma_output: the output tensor has %d channels, source format %d; luma frames are written from 1 channel with YUV chroma", t->c, src.format);
    SNNB_REQUIRE((src.format == SNNB_FRAME_P010) == (fr.format == SNNB_FRAME_P010), "launch_luma_output: source format %d, out format %d; P010 pairs with P010 only",
                 src.format, fr.format);
    const ChromaSource c = chroma_source(src.format);
    FrameV s {};
    s.w = src.width, s.h = src.height;
    for (int i = 0; i < 2; ++i)
        s.plane[1 + i] = src.plane[c.plane[i]] + c.offset[i], s.pitch[1 + i] = src.pitch[c.plane[i]], s.stride[1 + i] = src.image_stride[c.plane[i]];
    FrameOutV o;
    for (int i = 0; i < 3; ++i) o.plane[i] = fr.plane[i], o.pitch[i] = fr.pitch[i], o.stride[i] = fr.image_stride[i];
    o.w = fr.width, o.h = fr.height, o.scale = fr.scale, o.offset = fr.offset;
    const int linear = fr.linear_filter ? 1 : 0;
    const size_t blocks = (size_t) t->n * ((fr.height + 1) / 2) * ((fr.width + 1) / 2);
    const dim3 grid((unsigned) ((blocks + 255) / 256)), block(256);
    const int rc = with_format<FrameKernels::yuv>(fr.format, [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(luma_output_kernel<FMT>, grid, block, 0, ctx->stream, view(t), s, c.step, o, linear), "luma_output_kernel", format_name(FMT));
    });
    SNNB_REQUIRE(rc >= 0, "launch_luma_output: out format %d; luma frames are written as NV12, NV21, I420 or P010", fr.format);
    return rc;
}

// Model output 0 -> an 8-bit label plane (snnb_model_segment_frames): the fp32 scores hi + lo resampled to the plane with
// ImageTexture::resize's taps and blend_rn (step 2 of frame_output_kernel, on the scores rather than on quantised bytes), then one label
// per pixel: the arg-max over the C channels, or the threshold of a 1-channel output.
struct LabelsV {
    uint8_t* plane;
    int pitch;
    long long stride;
    int w, h;
    float threshold;
};
// The label of pixel (x, y) of image n. The channel loop reads 8 channels per load8 at each tap (1, or 4 when blending) and keeps only
// the running maximum and its index. THRESH: C == 1, no channel loop. Ties go to the lowest channel (strict >), NaN scores are never the
// maximum, and a pixel whose scores are all NaN is labelled 0.
template <bool THRESH>
__device__ __forceinline__ void segment_pixel(const TV& t, const LabelsV& o, int linear, int n, int x, int y) {
    const bool direct = o.w == t.W && o.h == t.H;
    ResizeTaps r;
    if (direct) r.x0 = r.x1 = x, r.y0 = r.y1 = y, r.ax = r.ay = 0.0f;
    else r = resize_taps(resize_pos(x, y, o.w, o.h, t.W, t.H), t.W, t.H, linear);
    const bool blend  = linear && !direct;
    const size_t img  = (size_t) n * t.H;
    const size_t o00 = ((img + r.y0) * t.W + r.x0) * t.Cp, o01 = ((img + r.y0) * t.W + r.x1) * t.Cp;
    const size_t o10 = ((img + r.y1) * t.W + r.x0) * t.Cp, o11 = ((img + r.y1) * t.W + r.x1) * t.Cp;
    int label;
    if (THRESH) {
        float p00[8];
        load8(t.hi, t.lo, o00, p00);
        float s = p00[0];
        if (blend) {
            float p01[8], p10[8], p11[8];
            load8(t.hi, t.lo, o01, p01);
            load8(t.hi, t.lo, o10, p10);
            load8(t.hi, t.lo, o11, p11);
            s = blend_rn(r, p00[0], p01[0], p10[0], p11[0]);
        }
        label = s >= o.threshold ? 1 : 0; // false for NaN
    } else {
        float best = -INFINITY;
        int arg    = -1;
#pragma unroll 1
        for (int c = 0; c < t.C; c += 8) {
            float s[8];
            load8(t.hi, t.lo, o00 + c, s);
            if (blend) {
                float p01[8], p10[8], p11[8];
                load8(t.hi, t.lo, o01 + c, p01);
                load8(t.hi, t.lo, o10 + c, p10);
                load8(t.hi, t.lo, o11 + c, p11);
#pragma unroll
                for (int j = 0; j < 8; ++j) s[j] = blend_rn(r, s[j], p01[j], p10[j], p11[j]);
            }
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (c + j < t.C && (s[j] > best || (arg < 0 && s[j] == s[j]))) best = s[j], arg = c + j;
        }
        label = arg < 0 ? 0 : arg;
    }
    o.plane[n * o.stride + (size_t) y * o.pitch + x] = (uint8_t) label;
}
// One thread per label pixel, x fastest: the pixels of a warp lie in one row and share their tap rows. A block covers SEG_THREADS
// pixels of a row (grid x); rows and images come from grid y and z, strided past 65535, so no thread divides.
constexpr int SEG_THREADS = 128;
template <bool THRESH>
__global__ void __launch_bounds__(SEG_THREADS) segment_output_kernel(TV t, LabelsV o, int linear) {
    pdl_wait();
    const int x = blockIdx.x * SEG_THREADS + threadIdx.x;
    if (x >= o.w) return;
    for (int n = blockIdx.z; n < t.N; n += gridDim.z)
        for (int y = blockIdx.y; y < o.h; y += gridDim.y) segment_pixel<THRESH>(t, o, linear, n, x, y);
}
int launch_segment_output(snnb_context* ctx, const snnb_tensor* t, const snnb_labels_out& lo) {
    SNNB_REQUIRE(t->c >= 1 && t->c <= 256 && t->cp % 8 == 0 && !t->feed_only, "launch_segment_output: the output tensor has %d channels; labels are written from 1 to 256",
                 t->c);
    LabelsV o;
    o.plane = lo.plane, o.pitch = lo.pitch, o.stride = lo.image_stride, o.w = lo.width, o.h = lo.height, o.threshold = lo.threshold;
    const int linear = lo.linear_filter ? 1 : 0;
    const dim3 grid((unsigned) ((lo.width + SEG_THREADS - 1) / SEG_THREADS), (unsigned) std::min(lo.height, 65535), (unsigned) std::min(t->n, 65535)),
        block(SEG_THREADS);
    if (t->c == 1) return launch_done(ctx, launch_k(segment_output_kernel<true>, grid, block, 0, ctx->stream, view(t), o, linear), "segment_output_kernel<threshold>");
    return launch_done(ctx, launch_k(segment_output_kernel<false>, grid, block, 0, ctx->stream, view(t), o, linear), "segment_output_kernel<argmax>");
}

// Output lists (snnb_model_transform_frame_list / transform_luma_list / segment_frame_list): slot n of the model's output 0 written to
// out image n, each image its own allocation and size. Each table is a __grid_constant__ parameter, as FrameListV, with compact entries
// (no image strides) so that the luma kernel's source chroma and destination tables for 256 images fit the 32,764-byte parameter limit
// together. The work per image differs (a 2160p image has 9x the 2 x 2 blocks of a 720p one), so the grid is the sum of each image's own
// CTA count: first[n] is image n's first CTA, and a CTA finds its image by a binary search on blockIdx.x. The search is uniform across
// the CTA, so its constant-bank reads broadcast. Inside the image, indexing is the batch kernel's, through the same per-pixel helpers,
// with slot n for the model tensor and image 0 (stride 0) for the planes.
struct OutImageV {
    uint8_t* plane[3];
    int pitch[3];
    int w, h;
};
struct ChromaImageV { // the source chroma of transform_luma_list: U and V as launch_luma_output's planes 1 and 2 of FrameV
    const uint8_t* u;
    const uint8_t* v;
    int pitch_u, pitch_v;
    int w, h; // the source frame's size
};
struct LabelsImageV {
    uint8_t* plane;
    int pitch;
    int w, h;
};
struct FrameOutListV {
    int count;
    unsigned first[SNNB_FRAME_LIST_MAX];
    OutImageV img[SNNB_FRAME_LIST_MAX];
};
struct ChromaListV {
    ChromaImageV img[SNNB_FRAME_LIST_MAX];
};
struct LabelsListV {
    int count;
    unsigned first[SNNB_FRAME_LIST_MAX];
    LabelsImageV img[SNNB_FRAME_LIST_MAX];
};
constexpr size_t KERNEL_PARAM_BYTES = 32764; // CUDA 12.1+ on Volta and later
static_assert(sizeof(FrameOutListV) <= KERNEL_PARAM_BYTES - sizeof(TV) - 3 * sizeof(float), "frame_list_output_kernel's parameters");
static_assert(sizeof(FrameOutListV) + sizeof(ChromaListV) <= KERNEL_PARAM_BYTES - sizeof(TV) - 4 * sizeof(float), "luma_list_output_kernel's parameters");
static_assert(sizeof(LabelsListV) <= KERNEL_PARAM_BYTES - sizeof(TV) - 2 * sizeof(float), "segment_list_output_kernel's parameters");

// The image of this CTA: the last n < count with first[n] <= blockIdx.x (first[0] = 0, strictly increasing)
__device__ __forceinline__ int list_image(const unsigned* first, int count) {
    int lo = 0, hi = count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (first[mid] <= blockIdx.x) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}
// 256 threads per CTA, one per 2 x 2 block of image n's output (frame_out_block)
template <int FMT>
__global__ void __launch_bounds__(256) frame_list_output_kernel(TV t, const __grid_constant__ FrameOutListV L, float scale, float offset, int linear) {
    pdl_wait();
    const int n         = list_image(L.first, L.count);
    const OutImageV& e  = L.img[n];
    const int cw = (e.w + 1) >> 1, ch = (e.h + 1) >> 1;
    const size_t gid = (size_t) (blockIdx.x - L.first[n]) * blockDim.x + threadIdx.x;
    if (gid >= (size_t) cw * ch) return;
    FrameOutV o;
#pragma unroll
    for (int p = 0; p < 3; ++p) o.plane[p] = e.plane[p], o.pitch[p] = e.pitch[p], o.stride[p] = 0;
    o.w = e.w, o.h = e.h, o.scale = scale, o.offset = offset;
    frame_out_block<FMT>(t, o, n, (int) (gid % cw), (int) (gid / cw), linear);
}
// As frame_list_output_kernel, with luma_out_block and image n's source chroma from S
template <int FMT>
__global__ void __launch_bounds__(256) luma_list_output_kernel(TV t, const __grid_constant__ FrameOutListV L, const __grid_constant__ ChromaListV S, int step,
                                                               float scale, float offset, int linear) {
    pdl_wait();
    const int n         = list_image(L.first, L.count);
    const OutImageV& e  = L.img[n];
    const int cw = (e.w + 1) >> 1, ch = (e.h + 1) >> 1;
    const size_t gid = (size_t) (blockIdx.x - L.first[n]) * blockDim.x + threadIdx.x;
    if (gid >= (size_t) cw * ch) return;
    FrameOutV o;
#pragma unroll
    for (int p = 0; p < 3; ++p) o.plane[p] = e.plane[p], o.pitch[p] = e.pitch[p], o.stride[p] = 0;
    o.w = e.w, o.h = e.h, o.scale = scale, o.offset = offset;
    const ChromaImageV& c = S.img[n];
    FrameV s {};
    s.plane[1] = c.u, s.plane[2] = c.v, s.pitch[1] = c.pitch_u, s.pitch[2] = c.pitch_v, s.w = c.w, s.h = c.h;
    luma_out_block<FMT>(t, s, step, o, n, (int) (gid % cw), (int) (gid / cw), linear);
}
// SEG_THREADS pixels of one row of image n's label plane per CTA, x fastest, as segment_output_kernel
template <bool THRESH>
__global__ void __launch_bounds__(SEG_THREADS) segment_list_output_kernel(TV t, const __grid_constant__ LabelsListV L, float threshold, int linear) {
    pdl_wait();
    const int n           = list_image(L.first, L.count);
    const LabelsImageV& e = L.img[n];
    const int row_ctas = (e.w + SEG_THREADS - 1) / SEG_THREADS;
    const int local    = (int) (blockIdx.x - L.first[n]);
    const int y = local / row_ctas, x = (local - y * row_ctas) * SEG_THREADS + threadIdx.x;
    if (x >= e.w) return;
    LabelsV o;
    o.plane = e.plane, o.pitch = e.pitch, o.stride = 0, o.w = e.w, o.h = e.h, o.threshold = threshold;
    segment_pixel<THRESH>(t, o, linear, n, x, y);
}

// first[] of a list whose image n takes ctas(n) CTAs; false when the grid would exceed 2^31 - 1 CTAs
template <typename F>
static bool list_grid(int count, unsigned first[], F ctas, unsigned& total) {
    long long sum = 0;
    for (int n = 0; n < count; ++n) {
        first[n] = (unsigned) sum;
        sum += ctas(n);
        if (sum > 0x7fffffffLL) return false;
    }
    total = (unsigned) sum;
    return true;
}
// The destination table of an output list (count == t->n <= SNNB_FRAME_LIST_MAX, checked by the caller), 256 threads per CTA, one per
// 2 x 2 block of each image
static int frame_out_list_view(const char* who, const snnb_tensor* t, const snnb_frame_out_list& fo, FrameOutListV& L, unsigned& grid) {
    SNNB_REQUIRE(fo.count == t->n && fo.count >= 1 && fo.count <= SNNB_FRAME_LIST_MAX, "%s: %d images for a batch of %d", who, fo.count, t->n);
    std::memset(&L, 0, sizeof(L));
    L.count = fo.count;
    for (int n = 0; n < fo.count; ++n) {
        const snnb_frame_out_image& im = fo.images[n];
        for (int p = 0; p < 3; ++p) L.img[n].plane[p] = im.plane[p], L.img[n].pitch[p] = im.pitch[p];
        L.img[n].w = im.width, L.img[n].h = im.height;
    }
    const bool fits = list_grid(fo.count, L.first, [&](int n) { return ((long long) ((L.img[n].h + 1) / 2) * ((L.img[n].w + 1) / 2) + 255) / 256; }, grid);
    SNNB_REQUIRE(fits, "%s: the list's output needs more than 2^31 - 1 CTAs", who);
    return 0;
}
int launch_frame_output(snnb_context* ctx, const snnb_tensor* t, const snnb_frame_out_list& fo) {
    SNNB_REQUIRE((t->c == 1 || t->c == 3 || t->c == 4) && t->cp == 8 && !t->feed_only,
                 "launch_frame_list_output: the output tensor has %d channels; frames are written from 1, 3 or 4", t->c);
    FrameOutListV L;
    unsigned blocks = 0;
    if (frame_out_list_view("launch_frame_list_output", t, fo, L, blocks)) return 1;
    const int linear = fo.linear_filter ? 1 : 0;
    const dim3 grid(blocks), block(256);
    const int rc = with_format<FrameKernels::all>(fo.format, [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(frame_list_output_kernel<FMT>, grid, block, 0, ctx->stream, view(t), L, fo.scale, fo.offset, linear),
                           "frame_list_output_kernel", format_name(FMT));
    });
    SNNB_REQUIRE(rc >= 0, "launch_frame_list_output: unknown format %d", fo.format);
    return rc;
}
int launch_luma_output(snnb_context* ctx, const snnb_tensor* t, const snnb_frame_list& src, const snnb_frame_out_list& fo) {
    SNNB_REQUIRE(t->c == 1 && t->cp == 8 && !t->feed_only && src.format != SNNB_FRAME_RGBA8,
                 "launch_luma_list_output: the output tensor has %d channels, source format %d; luma frames are written from 1 channel with YUV chroma", t->c,
                 src.format);
    SNNB_REQUIRE((src.format == SNNB_FRAME_P010) == (fo.format == SNNB_FRAME_P010),
                 "launch_luma_list_output: source format %d, out format %d; P010 pairs with P010 only", src.format, fo.format);
    SNNB_REQUIRE(src.count == fo.count, "launch_luma_list_output: %d source images for %d out images", src.count, fo.count);
    FrameOutListV L;
    unsigned blocks = 0;
    if (frame_out_list_view("launch_luma_list_output", t, fo, L, blocks)) return 1;
    const ChromaSource c = chroma_source(src.format);
    ChromaListV S;
    std::memset(&S, 0, sizeof(S));
    for (int n = 0; n < src.count; ++n) {
        const snnb_frame_image& im = src.images[n];
        S.img[n] = ChromaImageV {im.plane[c.plane[0]] + c.offset[0], im.plane[c.plane[1]] + c.offset[1], im.pitch[c.plane[0]], im.pitch[c.plane[1]], im.width,
                                 im.height};
    }
    const int linear = fo.linear_filter ? 1 : 0;
    const dim3 grid(blocks), block(256);
    const int rc = with_format<FrameKernels::yuv>(fo.format, [&](auto fmt) {
        constexpr int FMT = decltype(fmt)::value;
        return launch_done(ctx, launch_k(luma_list_output_kernel<FMT>, grid, block, 0, ctx->stream, view(t), L, S, c.step, fo.scale, fo.offset, linear),
                           "luma_list_output_kernel", format_name(FMT));
    });
    SNNB_REQUIRE(rc >= 0, "launch_luma_list_output: out format %d; luma frames are written as NV12, NV21, I420 or P010", fo.format);
    return rc;
}
int launch_segment_output(snnb_context* ctx, const snnb_tensor* t, const snnb_labels_list& lo) {
    SNNB_REQUIRE(t->c >= 1 && t->c <= 256 && t->cp % 8 == 0 && !t->feed_only,
                 "launch_segment_list_output: the output tensor has %d channels; labels are written from 1 to 256", t->c);
    SNNB_REQUIRE(lo.count == t->n && lo.count >= 1 && lo.count <= SNNB_FRAME_LIST_MAX, "launch_segment_list_output: %d images for a batch of %d", lo.count, t->n);
    LabelsListV L;
    std::memset(&L, 0, sizeof(L));
    L.count = lo.count;
    for (int n = 0; n < lo.count; ++n) L.img[n] = LabelsImageV {lo.images[n].plane, lo.images[n].pitch, lo.images[n].width, lo.images[n].height};
    unsigned blocks = 0;
    const bool fits = list_grid(lo.count, L.first, [&](int n) { return (long long) ((L.img[n].w + SEG_THREADS - 1) / SEG_THREADS) * L.img[n].h; }, blocks);
    SNNB_REQUIRE(fits, "launch_segment_list_output: the list's labels need more than 2^31 - 1 CTAs");
    const int linear = lo.linear_filter ? 1 : 0;
    const dim3 grid(blocks), block(SEG_THREADS);
    if (t->c == 1)
        return launch_done(ctx, launch_k(segment_list_output_kernel<true>, grid, block, 0, ctx->stream, view(t), L, lo.threshold, linear),
                           "segment_list_output_kernel<threshold>");
    return launch_done(ctx, launch_k(segment_list_output_kernel<false>, grid, block, 0, ctx->stream, view(t), L, lo.threshold, linear),
                       "segment_list_output_kernel<argmax>");
}

} // namespace snnb
