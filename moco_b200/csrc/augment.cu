// The two pre-training crops' augmentation on the GPU (moco_augment_crops, include/moco_b200.h).
//
// Reference: train.py:106-114 -- RandomResizedCrop(224) -> RandomGrayscale(0.2) -> ColorJitter(0.4, 0.4, 0.4, 0.4) ->
// RandomHorizontalFlip -> ToTensor -> Normalize, run twice per image by moco/dataset.py:25-33.  The random draws are
// made on the host (moco_b200/augment.py); each crop arrives here as a moco_aug_crop record and the kernels evaluate
// torchvision's TENSOR implementation of the same ops on decoded_uint8 / 255 in fp32:
//   resized_crop(antialias=True)  ATen's upsample_bilinear2d_aa: triangle filter of support max(scale, 1), taps
//                                 clipped at the crop's border, weights renormalised to sum 1.  Evaluated as a vertical
//                                 then a horizontal pass (ATen's CPU kernel runs horizontal first: the two differ by
//                                 fp32 rounding of the sums only).
//   rgb_to_grayscale              0.2989 r + 0.587 g + 0.114 b, left to right, each product rounded.
//   adjust_brightness / contrast / saturation / hue in the drawn order; _blend = clamp(ratio a + (1 - ratio) b, 0, 1);
//                                 the contrast mean is the mean grayscale of the whole crop as it stands before the
//                                 contrast op; hue through _rgb2hsv / _hsv2rgb with the shift taken % 1.0.
//   hflip                         folded into the store address: output column ox is computed from column W-1-ox.
//   Normalize                     (x - mean) / std, a subtraction then a division.
// Every operation is one IEEE fp32 operation rounded to nearest (no contraction into FMA), in torchvision's order.
//
// Two kernels.  The contrast mean depends on the whole crop, so aug_mean_kernel (one CTA per crop, fixed summation
// order) recomputes the resample and the ops before the contrast op and reduces the grayscale into crop_means[i];
// aug_apply_kernel then evaluates everything and stores.  Recomputing rather than staging: the fp32 intermediate of a
// 256-image batch would be 308 MB of extra traffic plus a buffer the caller would have to provide.
//
// One output row of one crop: the vertical pass reads the crop's source rows (contiguous uint8 HWC bytes, coalesced)
// into a shared fp32 row v[x][c]; the horizontal pass gives each thread one output pixel.  A crop wider than kAugSpan
// source pixels is processed in column chunks whose source span fits v.
//
// The MoCo v2 entry (moco_augment_crops_blur) runs the same two passes over its 128-byte records, with grayscale after
// the jitter where the record asks for it, and a third kernel for the blurred crops: aug_blur_kernel evaluates a band
// of up to kBlurRows output rows plus the blur's h rows either side through the same row pass into shared memory
// (fp32 RGB, unflipped), then blurs the band's rows out of it, one output row at a time: the vertical pass into the
// row buffer v, then the horizontal pass, the normalise and the (flipped) store.  Reflected rows never leave the band:
// a row above it is reflected only while y < h, so it lands in [0, h], inside [y0 - h, y0 + R + h); likewise below.
// Unblurred crops keep aug_apply_kernel's 8-row CTAs; each apply kernel's CTAs of the other kind exit at once.
//
// The validation transform (moco_resize_center_crops, eval.py:111-116: Resize -> CenterCrop -> Normalize) runs on the
// same row pass: its "crop" is the whole source image resampled to resized_h x resized_w, and only the output window
// [top, top + out_h) x [left, left + out_w) of that resized image is evaluated -- the window's origin is added to the
// tap index (AugCtx::oy0 / ox0), which is 0 for the pre-training crops.  One kernel, no pointwise ops.
#include "common.cuh"

namespace moco {

constexpr int kAugThreads = 256;
constexpr int kAugRows = 8;             // output rows per CTA of the apply pass
constexpr int kAugSpan = 2048;          // source pixels of one column chunk held in shared memory (24 KB of fp32 RGB)
constexpr int kAugMaxOut = 1024;        // largest out_h / out_w
constexpr int kBlurThreads = 512;
constexpr int kBlurMaxOut = 512;        // largest out_h / out_w of moco_augment_crops_blur
constexpr int kBlurRows = 32;           // output rows per CTA of the blur pass, at most
constexpr int kBlurMaxTaps = 31;
constexpr int kBlurBandBytes = 192 * 1024;   // the band's dynamic shared memory, at most

struct AugTap {                         // one output column's (or row's) taps: source [lo, lo + n), crop-relative
    int lo, n;
    float center, norm;                 // weight of tap j = filter(((lo + j) - center + 0.5) * invscale) * norm
};

// ATen's _compute_indices_min_size_weights_aa for the bilinear (triangle) filter, without storing the weights.
__device__ __forceinline__ AugTap aug_tap(int i, float scale, float support, float invscale, int in_size) {
    AugTap t;
    t.center = (float)((double)scale * (i + 0.5));
    const int max_n = (int)ceilf(support) * 2 + 1;
    const long long lo = max((long long)((double)(t.center - support) + 0.5), 0LL);
    const long long hi = min((long long)((double)(t.center + support) + 0.5), (long long)in_size);
    t.lo = (int)lo;
    t.n = (int)max(0LL, min(hi - lo, (long long)max_n));
    float total = 0.f;
    for (int j = 0; j < t.n; ++j) {
        const float x = fabsf(__fmul_rn(__fadd_rn(__fsub_rn((float)(t.lo + j), t.center), 0.5f), invscale));
        total = __fadd_rn(total, x < 1.f ? __fsub_rn(1.f, x) : 0.f);
    }
    t.norm = total != 0.f ? __frcp_rn(total) : 0.f;
    return t;
}

__device__ __forceinline__ float aug_weight(int k, const AugTap& t, float invscale) {
    const float x = fabsf(__fmul_rn(__fadd_rn(__fsub_rn((float)k, t.center), 0.5f), invscale));
    return x < 1.f ? __fmul_rn(__fsub_rn(1.f, x), t.norm) : 0.f;
}

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.f), 1.f); }

__device__ __forceinline__ float gray(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// _blend(a, b, ratio) with one_minus = fp32(1.0 - ratio)
__device__ __forceinline__ float blend(float a, float b, float ratio, float one_minus) {
    return clamp01(__fadd_rn(__fmul_rn(ratio, a), __fmul_rn(one_minus, b)));
}

// adjust_hue: _rgb2hsv, h = (h + hue) % 1.0, _hsv2rgb
__device__ __forceinline__ void hue_shift(float& r, float& g, float& b, float hue) {
    const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
    const bool eqc = maxc == minc;
    const float cr = __fsub_rn(maxc, minc);
    const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
    const float crd = eqc ? 1.f : cr;
    const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd);
    const float gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
    const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
    const float hr = (maxc == r) ? __fsub_rn(bc, gc) : 0.f;
    const float hg = (maxc == g && maxc != r) ? __fsub_rn(__fadd_rn(2.f, rc), bc) : 0.f;
    const float hb = (maxc != g && maxc != r) ? __fsub_rn(__fadd_rn(4.f, gc), rc) : 0.f;
    float h = fmodf(__fadd_rn(__fdiv_rn(__fadd_rn(__fadd_rn(hr, hg), hb), 6.f), 1.f), 1.f);
    h = fmodf(__fadd_rn(h, hue), 1.f);                      // torch.remainder: the sign of the divisor
    if (h != 0.f && h < 0.f) h = __fadd_rn(h, 1.f);
    const float v = maxc;
    const float h6 = __fmul_rn(h, 6.f);
    const float fi = floorf(h6);
    const float f = __fsub_rn(h6, fi);
    const int i = ((int)fi % 6 + 6) % 6;
    const float p = clamp01(__fmul_rn(v, __fsub_rn(1.f, s)));
    const float q = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, f))));
    const float t = clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, f)))));
    switch (i) {
        case 0: r = v; g = t; b = p; break;
        case 1: r = q; g = v; b = p; break;
        case 2: r = p; g = v; b = t; break;
        case 3: r = p; g = q; b = v; break;
        case 4: r = t; g = p; b = v; break;
        default: r = v; g = p; b = q; break;
    }
}

// One crop's record, clamped so that every source index stays inside its image and inside the pixel buffer.
struct AugCtx {
    const uint8_t* pix;
    unsigned long long last;            // pixels_bytes - 1
    unsigned long long base;            // byte index of the crop's top-left pixel
    unsigned long long row_bytes;       // src_w * 3
    int hh, ww;                         // crop box size
    int oy0, ox0;                       // tap index of output row / column 0 (the resize window's top, left)
    int flags, order, cw;               // cw: output columns per chunk
    bool gray_late, blur;               // moco_aug_crop_blur's switches (false for the other records)
    float sy, supy, invy, sx, supx, invx;
    float f[4], fm[4];                  // brightness, contrast, saturation, hue; fm[k] = fp32(1.0 - f[k])
};

// The resample of the c.hh x c.ww box to dst_h x dst_w (ATen's scale = in / out), of which out_w columns are computed.
__device__ void aug_scales(AugCtx& c, int dst_h, int dst_w, int out_w) {
    c.sy = (float)c.hh / (float)dst_h;
    c.sx = (float)c.ww / (float)dst_w;
    c.supy = c.sy >= 1.f ? c.sy : 1.f;
    c.supx = c.sx >= 1.f ? c.sx : 1.f;
    c.invy = c.sy >= 1.f ? (float)(1.0 / (double)c.sy) : 1.f;
    c.invx = c.sx >= 1.f ? (float)(1.0 / (double)c.sx) : 1.f;
    c.cw = out_w;
    if (c.ww > kAugSpan) c.cw = max(1, min(out_w, (int)((float)(kAugSpan - 4) / c.sx) - 1));
}

__device__ AugCtx aug_ctx(const uint8_t* pix, unsigned long long pixels_bytes, const moco_aug_crop& cr, int out_h,
                          int out_w) {
    AugCtx c;
    c.pix = pix;
    c.last = pixels_bytes - 1;
    const int H = max(cr.src_h, 1), W = max(cr.src_w, 1);
    const int top = min(max(cr.top, 0), H - 1), left = min(max(cr.left, 0), W - 1);
    c.hh = min(max(cr.height, 1), H - top);
    c.ww = min(max(cr.width, 1), W - left);
    const unsigned long long off = cr.src_offset < 0 ? 0ULL : (unsigned long long)cr.src_offset;
    c.row_bytes = (unsigned long long)W * 3ULL;
    c.base = off + (unsigned long long)top * c.row_bytes + (unsigned long long)left * 3ULL;
    c.oy0 = c.ox0 = 0;
    c.flags = cr.flags;
    c.order = cr.order;
    c.gray_late = c.blur = false;
    aug_scales(c, out_h, out_w, out_w);
    const float fs[4] = {cr.brightness, cr.contrast, cr.saturation, cr.hue};
#pragma unroll
    for (int k = 0; k < 4; ++k) { c.f[k] = fs[k]; c.fm[k] = (float)(1.0 - (double)fs[k]); }
    return c;
}

// The pointwise ops of one pixel.  Stop at the contrast op (returning false) when mean == nullptr, the reduction pass.
__device__ __forceinline__ bool aug_pointwise(const AugCtx& c, float& r, float& g, float& b, const float* mean) {
    const bool gray_op = c.flags & MOCO_AUG_GRAY;
    if (gray_op && !c.gray_late) { const float l = gray(r, g, b); r = g = b = l; }
    if (!(c.flags & MOCO_AUG_JITTER)) {
        if (gray_op && c.gray_late) { const float l = gray(r, g, b); r = g = b = l; }
        return true;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int op = (c.order >> (2 * k)) & 3;
        if (op == 0) {
            r = blend(r, 0.f, c.f[0], c.fm[0]); g = blend(g, 0.f, c.f[0], c.fm[0]); b = blend(b, 0.f, c.f[0], c.fm[0]);
        } else if (op == 1) {
            if (!mean) return false;
            const float m = *mean;
            r = blend(r, m, c.f[1], c.fm[1]); g = blend(g, m, c.f[1], c.fm[1]); b = blend(b, m, c.f[1], c.fm[1]);
        } else if (op == 2) {
            const float l = gray(r, g, b);
            r = blend(r, l, c.f[2], c.fm[2]); g = blend(g, l, c.f[2], c.fm[2]); b = blend(b, l, c.f[2], c.fm[2]);
        } else {
            hue_shift(r, g, b, c.f[3]);
        }
    }
    if (gray_op && c.gray_late) { const float l = gray(r, g, b); r = g = b = l; }
    return true;
}

struct AugOut {                         // the apply pass's destination (dst and band nullptr: the reduction pass)
    void* dst;
    int dtype;
    long long plane;                    // out_h * out_w
    const float* norm;                  // mean[3], std[3]
    const float* mean;                  // the crop's contrast mean
    float* band;                        // the blur pass: row oy's pixel x at band[((oy - band_y0) * out_w + x) * 3]
    int band_y0;
};

// Normalise and store output pixel (oy, ox) of crop `crop`.
__device__ __forceinline__ void aug_store(const AugOut& o, long long crop, int oy, int ox, int out_w, float r, float g,
                                          float b) {
    const long long at = crop * 3 * o.plane + (long long)oy * out_w + ox;
    const float val[3] = {__fdiv_rn(__fsub_rn(r, o.norm[0]), o.norm[3]),
                          __fdiv_rn(__fsub_rn(g, o.norm[1]), o.norm[4]),
                          __fdiv_rn(__fsub_rn(b, o.norm[2]), o.norm[5])};
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        if (o.dtype == MOCO_BF16)
            static_cast<__nv_bfloat16*>(o.dst)[at + ch * o.plane] = __float2bfloat16_rn(val[ch]);
        else
            static_cast<float*>(o.dst)[at + ch * o.plane] = val[ch];
    }
}

// One output row oy: resample, pointwise ops, then either store (o.dst), write the band (o.band) or add the grayscale
// of the pre-contrast value to gsum.  xt: the crop's column taps.  All threads of the CTA call it.
__device__ void aug_row(const AugCtx& c, const AugTap* xt, float* v, int oy, int out_w, const AugOut& o,
                        long long crop, float& gsum) {
    const AugTap ty = aug_tap(c.oy0 + oy, c.sy, c.supy, c.invy, c.hh);
    for (int a = 0; a < out_w; a += c.cw) {
        const int e = min(a + c.cw, out_w);
        const int x0 = xt[a].lo;
        const int n3 = min(xt[e - 1].lo + xt[e - 1].n - x0, kAugSpan) * 3;
        for (int k = threadIdx.x; k < n3; k += blockDim.x) {
            const unsigned long long col = c.base + (unsigned long long)x0 * 3ULL + (unsigned long long)k;
            float acc = 0.f;
            for (int j = 0; j < ty.n; ++j) {
                const int y = min(ty.lo + j, c.hh - 1);
                const unsigned long long idx = min(col + (unsigned long long)y * c.row_bytes, c.last);
                acc = __fadd_rn(acc, __fmul_rn(aug_weight(ty.lo + j, ty, c.invy), (float)__ldg(c.pix + idx)));
            }
            v[k] = __fdiv_rn(acc, 255.f);
        }
        __syncthreads();
        for (int sx = a + threadIdx.x; sx < e; sx += blockDim.x) {
            const AugTap t = xt[sx];
            float r = 0.f, g = 0.f, b = 0.f;
            for (int j = 0; j < t.n; ++j) {
                const float w = aug_weight(t.lo + j, t, c.invx);
                const int i = min(max(t.lo + j - x0, 0), kAugSpan - 1) * 3;
                r = __fadd_rn(r, __fmul_rn(w, v[i]));
                g = __fadd_rn(g, __fmul_rn(w, v[i + 1]));
                b = __fadd_rn(b, __fmul_rn(w, v[i + 2]));
            }
            if (!o.dst && !o.band) {
                if (!aug_pointwise(c, r, g, b, nullptr)) gsum = __fadd_rn(gsum, gray(r, g, b));
                continue;
            }
            aug_pointwise(c, r, g, b, o.mean);
            if (o.band) {
                float* px = o.band + ((long long)(oy - o.band_y0) * out_w + sx) * 3;
                px[0] = r; px[1] = g; px[2] = b;
                continue;
            }
            aug_store(o, crop, oy, (c.flags & MOCO_AUG_FLIP) ? out_w - 1 - sx : sx, out_w, r, g, b);
        }
        __syncthreads();
    }
}

struct AugArgs {
    const uint8_t* pix;
    unsigned long long pixels_bytes;
    const char* recs;                   // record i at recs + i * rec_bytes: a moco_aug_crop or a moco_aug_crop_blur
    int rec_bytes;
    int out_h, out_w;
    int h, band_rows;                   // the blur pass: ksize / 2 and output rows per CTA
    float norm[6];
    void* dst;
    int dtype;
    float* means;
};

// Record i's context, with moco_aug_crop_blur's switches when the records are of that kind.
__device__ AugCtx aug_ctx_at(const AugArgs& p, int i) {
    const char* rec = p.recs + (long long)i * p.rec_bytes;
    AugCtx c = aug_ctx(p.pix, p.pixels_bytes, *reinterpret_cast<const moco_aug_crop*>(rec), p.out_h, p.out_w);
    if (p.rec_bytes == (int)sizeof(moco_aug_crop_blur)) {
        const moco_aug_crop_blur& rb = *reinterpret_cast<const moco_aug_crop_blur*>(rec);
        c.gray_late = rb.gray_after_jitter != 0;
        c.blur = rb.blur != 0;
    }
    return c;
}

__device__ void aug_columns(const AugCtx& c, AugTap* xt, int out_w) {
    for (int i = threadIdx.x; i < out_w; i += blockDim.x) xt[i] = aug_tap(c.ox0 + i, c.sx, c.supx, c.invx, c.ww);
    __syncthreads();
}

// the contrast mean of crop blockIdx.x (0 when its jitter is off)
__global__ void __launch_bounds__(kAugThreads) aug_mean_kernel(const __grid_constant__ AugArgs p) {
    __shared__ AugTap xt[kAugMaxOut];
    __shared__ float v[kAugSpan * 3];
    __shared__ float red[kAugThreads / 32];
    const AugCtx c = aug_ctx_at(p, blockIdx.x);
    if (!(c.flags & MOCO_AUG_JITTER)) {
        if (threadIdx.x == 0) p.means[blockIdx.x] = 0.f;
        return;
    }
    aug_columns(c, xt, p.out_w);
    const AugOut o = {nullptr, 0, 0, nullptr, nullptr, nullptr, 0};
    float gsum = 0.f;
    for (int oy = 0; oy < p.out_h; ++oy) aug_row(c, xt, v, oy, p.out_w, o, blockIdx.x, gsum);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) gsum = __fadd_rn(gsum, __shfl_xor_sync(0xffffffffu, gsum, s));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = gsum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int w = 0; w < kAugThreads / 32; ++w) s = __fadd_rn(s, red[w]);
        p.means[blockIdx.x] = __fdiv_rn(s, (float)((long long)p.out_h * p.out_w));
    }
}

// rows [blockIdx.x * kAugRows, +kAugRows) of crop blockIdx.y, unless it is blurred
__global__ void __launch_bounds__(kAugThreads) aug_apply_kernel(const __grid_constant__ AugArgs p) {
    __shared__ AugTap xt[kAugMaxOut];
    __shared__ float v[kAugSpan * 3];
    const AugCtx c = aug_ctx_at(p, blockIdx.y);
    if (c.blur) return;
    aug_columns(c, xt, p.out_w);
    const AugOut o = {p.dst, p.dtype, (long long)p.out_h * p.out_w, p.norm, p.means + blockIdx.y, nullptr, 0};
    float unused = 0.f;
    const int y1 = min((int)(blockIdx.x + 1) * kAugRows, p.out_h);
    for (int oy = blockIdx.x * kAugRows; oy < y1; ++oy) aug_row(c, xt, v, oy, p.out_w, o, blockIdx.y, unused);
}

__device__ __forceinline__ int reflect(int i, int n) {
    i = i < 0 ? -i : i;
    i = i >= n ? 2 * (n - 1) - i : i;
    return min(max(i, 0), n - 1);
}

// rows [blockIdx.x * band_rows, +band_rows) of crop blockIdx.y, if it is blurred: steps 1-4 of the band's rows and
// the h rows either side (clipped to the crop) into the dynamic shared memory, then the blur, one output row at a time
__global__ void __launch_bounds__(kBlurThreads) aug_blur_kernel(const __grid_constant__ AugArgs p) {
    extern __shared__ float band[];     // rows [lo, hi) of the crop after step 4, [row][x][rgb] fp32
    __shared__ AugTap xt[kBlurMaxOut];
    __shared__ float v[kAugSpan * 3];   // the row pass's resample row, then the blur's vertical pass of one row
    __shared__ float kw[kBlurMaxTaps];  // the full 1-D kernel, k[j] = weights[|j - h|]
    const AugCtx c = aug_ctx_at(p, blockIdx.y);
    if (!c.blur) return;
    const int h = p.h, out_h = p.out_h, out_w = p.out_w;
    const moco_aug_crop_blur& rb = reinterpret_cast<const moco_aug_crop_blur*>(p.recs)[blockIdx.y];
    if ((int)threadIdx.x <= 2 * h) kw[threadIdx.x] = rb.weights[abs((int)threadIdx.x - h)];
    aug_columns(c, xt, out_w);
    const int y0 = blockIdx.x * p.band_rows, y1 = min(y0 + p.band_rows, out_h);
    const int lo = max(y0 - h, 0), hi = min(y1 + h, out_h);
    const AugOut o = {p.dst, p.dtype, (long long)out_h * out_w, p.norm, p.means + blockIdx.y, band, lo};
    float unused = 0.f;
    for (int oy = lo; oy < hi; ++oy) aug_row(c, xt, v, oy, out_w, o, blockIdx.y, unused);   // ends with a barrier
    const bool flip = c.flags & MOCO_AUG_FLIP;
    for (int y = y0; y < y1; ++y) {
        for (int k = threadIdx.x; k < out_w * 3; k += blockDim.x) {
            const int x = k / 3, ch = k - 3 * x;
            float t = 0.f;
            for (int j = 0; j <= 2 * h; ++j) {
                const int row = min(max(reflect(y - h + j, out_h) - lo, 0), hi - lo - 1);
                t = __fadd_rn(t, __fmul_rn(kw[j], band[((long long)row * out_w + x) * 3 + ch]));
            }
            v[k] = t;
        }
        __syncthreads();
        for (int x = threadIdx.x; x < out_w; x += blockDim.x) {
            float s[3] = {0.f, 0.f, 0.f};
            for (int j = 0; j <= 2 * h; ++j) {
                const float w = kw[j];
                const int col = reflect(x - h + j, out_w) * 3;
#pragma unroll
                for (int ch = 0; ch < 3; ++ch) s[ch] = __fadd_rn(s[ch], __fmul_rn(w, v[col + ch]));
            }
            aug_store(o, blockIdx.y, y, flip ? out_w - 1 - x : x, out_w, s[0], s[1], s[2]);
        }
        __syncthreads();
    }
}

bool augment_shape_ok(int n_crops, int out_h, int out_w) {
    return n_crops >= 0 && n_crops <= 65535 && out_h >= 1 && out_h <= kAugMaxOut && out_w >= 1 && out_w <= kAugMaxOut;
}

// The blur pass's output rows per CTA: kBlurRows, or fewer where the band and its halo would not fit kBlurBandBytes,
// spread evenly over the crop's rows.  0: ksize or the size is outside moco_augment_crops_blur's envelope.
static int blur_band_rows(int out_h, int out_w, int ksize) {
    const int h = ksize / 2;
    if (ksize < 3 || ksize > kBlurMaxTaps || ksize % 2 == 0 || out_h < 1 || out_h > kBlurMaxOut || out_w < 1 ||
        out_w > kBlurMaxOut || h >= min(out_h, out_w))
        return 0;
    const int rows = min(kBlurRows, kBlurBandBytes / (out_w * 12) - 2 * h);
    if (rows < 1) return 0;
    const int bands = (out_h + rows - 1) / rows;
    return (out_h + bands - 1) / bands;
}

bool augment_blur_shape_ok(int n_crops, int out_h, int out_w, int ksize) {
    return n_crops >= 0 && n_crops <= 65535 && blur_band_rows(out_h, out_w, ksize) > 0;
}

static cudaError_t launch_aug(const void* pixels, size_t pixels_bytes, const void* recs, int rec_bytes, int n_crops,
                              int out_h, int out_w, int ksize, const float norm[6], void* dst, int dst_dtype,
                              float* crop_means, cudaStream_t stream) {
    if (n_crops == 0) return cudaSuccess;
    AugArgs p;
    p.pix = static_cast<const uint8_t*>(pixels);
    p.pixels_bytes = pixels_bytes;
    p.recs = static_cast<const char*>(recs);
    p.rec_bytes = rec_bytes;
    p.out_h = out_h;
    p.out_w = out_w;
    p.h = ksize / 2;
    p.band_rows = ksize ? blur_band_rows(out_h, out_w, ksize) : 0;
    for (int k = 0; k < 6; ++k) p.norm[k] = norm[k];
    p.dst = dst;
    p.dtype = dst_dtype;
    p.means = crop_means;
    aug_mean_kernel<<<n_crops, kAugThreads, 0, stream>>>(p);
    cudaError_t e = launched();
    if (e != cudaSuccess) return e;
    aug_apply_kernel<<<dim3((out_h + kAugRows - 1) / kAugRows, n_crops), kAugThreads, 0, stream>>>(p);
    e = launched();
    if (e != cudaSuccess || !ksize) return e;
    const int band_bytes = min(p.band_rows + 2 * p.h, out_h) * out_w * 12;
    e = cudaFuncSetAttribute(aug_blur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, band_bytes);
    if (e != cudaSuccess) return e;
    aug_blur_kernel<<<dim3((out_h + p.band_rows - 1) / p.band_rows, n_crops), kBlurThreads, band_bytes, stream>>>(p);
    return launched();
}

cudaError_t launch_augment(const void* pixels, size_t pixels_bytes, const moco_aug_crop* crops, int n_crops, int out_h,
                           int out_w, const float norm[6], void* dst, int dst_dtype, float* crop_means,
                           cudaStream_t stream) {
    if (!augment_shape_ok(n_crops, out_h, out_w)) return cudaErrorNotSupported;
    return launch_aug(pixels, pixels_bytes, crops, (int)sizeof(moco_aug_crop), n_crops, out_h, out_w, 0, norm, dst,
                      dst_dtype, crop_means, stream);
}

cudaError_t launch_augment_blur(const void* pixels, size_t pixels_bytes, const moco_aug_crop_blur* crops, int n_crops,
                                int out_h, int out_w, int ksize, const float norm[6], void* dst, int dst_dtype,
                                float* crop_means, cudaStream_t stream) {
    if (!augment_blur_shape_ok(n_crops, out_h, out_w, ksize)) return cudaErrorNotSupported;
    return launch_aug(pixels, pixels_bytes, crops, (int)sizeof(moco_aug_crop_blur), n_crops, out_h, out_w, ksize, norm,
                      dst, dst_dtype, crop_means, stream);
}

// One resize window's record, clamped like aug_ctx: the box is the whole source image, the resized size is at least
// the output's and the window lies inside the resized image, so every tap index stays inside the image.
__device__ AugCtx window_ctx(const uint8_t* pix, unsigned long long pixels_bytes, const moco_resize_window& wr,
                             int out_h, int out_w) {
    AugCtx c;
    c.pix = pix;
    c.last = pixels_bytes - 1;
    c.hh = max(wr.src_h, 1);
    c.ww = max(wr.src_w, 1);
    const unsigned long long off = wr.src_offset < 0 ? 0ULL : (unsigned long long)wr.src_offset;
    c.row_bytes = (unsigned long long)c.ww * 3ULL;
    c.base = off;
    const int rh = max(wr.resized_h, out_h), rw = max(wr.resized_w, out_w);
    c.oy0 = min(max(wr.top, 0), rh - out_h);
    c.ox0 = min(max(wr.left, 0), rw - out_w);
    c.flags = 0;
    c.order = 0;
    c.gray_late = c.blur = false;
    aug_scales(c, rh, rw, out_w);
#pragma unroll
    for (int k = 0; k < 4; ++k) { c.f[k] = 0.f; c.fm[k] = 1.f; }
    return c;
}

struct ResizeArgs {
    const uint8_t* pix;
    unsigned long long pixels_bytes;
    const moco_resize_window* windows;
    int out_h, out_w;
    float norm[6];
    void* dst;
    int dtype;
};

// rows [blockIdx.x * kAugRows, +kAugRows) of window blockIdx.y
__global__ void __launch_bounds__(kAugThreads) resize_window_kernel(const __grid_constant__ ResizeArgs p) {
    __shared__ AugTap xt[kAugMaxOut];
    __shared__ float v[kAugSpan * 3];
    const AugCtx c = window_ctx(p.pix, p.pixels_bytes, p.windows[blockIdx.y], p.out_h, p.out_w);
    aug_columns(c, xt, p.out_w);
    const AugOut o = {p.dst, p.dtype, (long long)p.out_h * p.out_w, p.norm, nullptr, nullptr, 0};
    float unused = 0.f;
    const int y1 = min((int)(blockIdx.x + 1) * kAugRows, p.out_h);
    for (int oy = blockIdx.x * kAugRows; oy < y1; ++oy) aug_row(c, xt, v, oy, p.out_w, o, blockIdx.y, unused);
}

cudaError_t launch_resize_windows(const void* pixels, size_t pixels_bytes, const moco_resize_window* windows, int n,
                                  int out_h, int out_w, const float norm[6], void* dst, int dst_dtype,
                                  cudaStream_t stream) {
    if (!augment_shape_ok(n, out_h, out_w)) return cudaErrorNotSupported;
    if (n == 0) return cudaSuccess;
    ResizeArgs p;
    p.pix = static_cast<const uint8_t*>(pixels);
    p.pixels_bytes = pixels_bytes;
    p.windows = windows;
    p.out_h = out_h;
    p.out_w = out_w;
    for (int k = 0; k < 6; ++k) p.norm[k] = norm[k];
    p.dst = dst;
    p.dtype = dst_dtype;
    resize_window_kernel<<<dim3((out_h + kAugRows - 1) / kAugRows, n), kAugThreads, 0, stream>>>(p);
    return launched();
}

}  // namespace moco
