// Convolution planning: which kernel runs a convolution, whether it reads a pre-padded copy of its input and whether a model
// input gets the compact 4-channel feed copy - decided here and nowhere else, from plain facts (ConvQuery, snnb_internal.h).
// The launchers only run what the plan names.
#include <algorithm>

#include "snnb_internal.h"

namespace snnb {

// Small-channel stems: IC <= 8 (one 16-byte vector per pixel), at most RW_MAX_N output channels, <= 8 K steps per filter row.
bool rowwin_packable(int in_c, int out_c, int k, int stride, int pad_x, RowPlan& rp) {
    return in_c <= 8 && out_c <= RW_MAX_N && make_row_plan(k, stride, pad_x, rp);
}

// Stride-2 stems with <= 4 input channels whose window fits the feed layout; they carry the row-window operand too.
bool feed_packable(int in_c, int out_c, int k, int stride, int pad_x, FeedPlan& fp) {
    RowPlan rp;
    return rowwin_packable(in_c, out_c, k, stride, pad_x, rp) && make_feed_plan(k, stride, pad_x, in_c, fp) && (254 + 2 * fp.nch) * 8 <= RW_ARR_BYTES;
}

// The row-window kernel takes the layer: its weights carry the operand for exactly this (stride, pad_x), no residual is fused, and
// the whole weight panel set stays resident in shared memory in the layout the launch uses (feed mode: fewer, shared rows).
static bool rowwin_fits(const ConvQuery& q, bool feed, const FeedPlan& fp, RowPlan& rp) {
    if (q.residual || q.row_stride != q.stride || q.row_pad != q.pad_x || !rowwin_packable(q.in_c, q.out_c, q.k, q.stride, q.pad_x, rp) ||
        UM_BLOCK_M + rp.span > RW_BOXW)
        return false;
    const int wrows = feed ? (q.k + fp.rows_per_panel - 1) / fp.rows_per_panel : q.k * ((rp.ksteps + 3) / 4); // 128-byte weight rows per channel
    return wrows * 2 * rowwin_nblk(q.out_c) * 128 <= RW_B_MAX_BYTES;
}

// The implicit GEMM: stride 1 or 2 (the TMA traversal stride on W and H), at least 16 input channels (below that K would be
// mostly zero padding), k <= 11, pads a TMA box coordinate can hold.
static bool igemm_fits(const ConvQuery& q) {
    return (q.stride == 1 || q.stride == 2) && q.in_c >= 16 && q.k >= 1 && q.k <= 11 && q.pad_x <= 127 && q.pad_y <= 127;
}

ConvPlan plan_conv(const ConvQuery& q) {
    ConvPlan p;
    p.pad_x = q.pad_x, p.pad_y = q.pad_y, p.pad_mode = q.pad_mode;
    if (q.algo == SNNB_ALGO_SIMT) return p;
    const int no_tensor = q.algo == SNNB_ALGO_AUTO ? CONV_SIMT : CONV_REFUSED;
    const FeedPlan no_feed;
    if (!(q.pad_mode == SNNB_PAD_NONE || q.pad_mode == SNNB_PAD_CONSTANT)) {
        // The TMA unit only zero-fills: replicate / reflect padding takes the tensor path on a pre-padded copy of the input, read
        // with zero padding. A fused residual rules out only the row-window kernel; the implicit GEMM then takes any channel count.
        ConvQuery padded = q;
        padded.pad_x = padded.pad_y = 0, padded.pad_mode = SNNB_PAD_CONSTANT, padded.residual = false;
        if (!q.may_prepad || q.k <= 1 || !(rowwin_fits(padded, false, no_feed, p.rp) || igemm_fits(padded))) {
            p.path = no_tensor;
            return p;
        }
        padded.residual = q.residual;
        p.pad_x = p.pad_y = 0, p.pad_mode = SNNB_PAD_CONSTANT;
        p.prepad_h = (q.out_h - 1) * q.stride + q.k; // the window of the last output pixel ends at (O - 1) s + k - 1 in padded coordinates
        p.prepad_w = (q.out_w - 1) * q.stride + q.k;
        p.path     = rowwin_fits(padded, false, no_feed, p.rp) ? CONV_ROWWIN : CONV_IGEMM;
        return p;
    }
    // FEED mode: a stride-2 RGB stem reading a model input, weights packed for this pad
    if (q.may_feed && !q.residual && q.feed_pad == q.pad_x && feed_packable(q.in_c, q.out_c, q.k, q.stride, q.pad_x, p.fp) && rowwin_fits(q, true, p.fp, p.rp)) {
        p.path = CONV_ROWWIN_FEED;
        // the copy holds every pixel the last tile's window segments touch: image pixel (y, x) at (y + pad_y, x + px)
        const int tiles_x = (q.out_w + UM_BLOCK_M - 1) / UM_BLOCK_M;
        const int need_w  = 2 * (tiles_x * UM_BLOCK_M - 1) + 2 * p.fp.nch;
        const int need_h  = 2 * (q.out_h - 1) + q.k;
        p.feed_w  = (std::max(q.in_w + p.fp.px, need_w) + 1) & ~1;
        p.feed_h  = std::max(q.in_h + q.pad_y, need_h);
        p.feed_py = q.pad_y, p.feed_px = p.fp.px;
        return p;
    }
    p.fp = no_feed;
    if (rowwin_fits(q, false, no_feed, p.rp))
        p.path = CONV_ROWWIN;
    else
        p.path = igemm_fits(q) ? CONV_IGEMM : no_tensor;
    return p;
}

int launch_conv2d(snnb_context* ctx, const ConvArgs& a, const ConvPlan& plan) {
    switch (plan.path) {
    case CONV_SIMT: return launch_conv2d_simt(ctx, a);
    case CONV_IGEMM: return launch_conv2d_umma(ctx, a);
    case CONV_ROWWIN:
    case CONV_ROWWIN_FEED: return launch_conv2d_rowwin(ctx, a, plan);
    }
    set_error("tensor-core path requested but unsupported for this shape (IC=%d OC=%d k=%d s=%d pad_mode=%d)", a.in->c, a.out->c, a.k, a.stride, a.pad_mode);
    return 2;
}

int launch_dense(snnb_context* ctx, const snnb_tensor* in, snnb_tensor* flat, snnb_tensor* out, const snnb_weights* w, int act, float alpha, int precision) {
    const snnb_tensor* x = in;
    if (in->h * in->w != 1) { // CPU Flatten order = HWC (cpulayer.h:94-115)
        if (launch_flatten(ctx, in, flat)) return 1;
        x = flat;
    }
    const bool softmax = act == SNNB_ACT_SOFTMAX;
    ConvQuery q;
    q.in_h = q.in_w = q.out_h = q.out_w = 1;
    q.in_c = x->c, q.out_c = out->c;
    q.row_stride = w->row_stride, q.row_pad = w->row_pad, q.feed_pad = w->feed_pad;
    ConvArgs a {x, nullptr, out, w, 1, 1, 0, 0, SNNB_PAD_NONE, softmax ? SNNB_ACT_NONE : act, alpha};
    a.precision = precision;
    // SiLU on the CPU Dense path is a by-value no-op in the reference (cpulayer.h:245-252); we apply the real SiLU (SURVEY Q10).
    if (launch_conv2d(ctx, a, plan_conv(q))) return 1;
    return softmax ? launch_softmax(ctx, out, out) : 0;
}

} // namespace snnb
