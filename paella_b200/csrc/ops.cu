// Memory-bound kernels of the denoiser (all channels-last, fp32 residual stream, fp16 GEMM operands).
//   embed_tokens   in_mapper (Embedding + LayerNorm) + PixelUnshuffle      ref/src/modules.py:126-131,271
//   ln_rows        LayerNorm2d / nn.LayerNorm(no affine, eps 1e-6)         ref/src/modules.py:22-27,125
//   ln_patchify2   LayerNorm2d + the im2col of Conv2d(k=2,s=2)             ref/src/modules.py:153-156
//   dwconv_ln      ResBlock.depthwise (+cat skip, groups=c) + LayerNorm2d  ref/src/modules.py:46-47,57-60
//   grn_*          GlobalResponseNorm                                      ref/src/modules.py:30-40
//   r_embed / film gen_r_embedding + TimestepBlock.mapper                  ref/src/modules.py:212-221,99-106
//   silu_cast      AttnBlock.kv_mapper's SiLU                              ref/src/modules.py:71-74
#include "ops.cuh"
#include "attention.cuh"

namespace pb {

constexpr float LN_EPS = 1e-6f;

__device__ __forceinline__ float ln_rstd(float var) { return 1.0f / sqrtf(var + LN_EPS); }

// ------------------------------------------------------------------ embed_tokens
// one warp per output row (b, y2, x2); row staged in shared memory so the global store is contiguous
__global__ void __launch_bounds__(256) embed_tokens_kernel(const int64_t* __restrict__ tokens, const float* __restrict__ emb,
                                                           int num_labels, int c_in, int B, int H, int W, int ps,
                                                           __half* __restrict__ out) {
    extern __shared__ __half s_row[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int h2 = H / ps, w2 = W / ps;
    const int64_t orow = (int64_t)blockIdx.x * 8 + warp;
    const int rowlen = c_in * ps * ps;
    __half* srow = s_row + warp * rowlen;
    if (orow < (int64_t)B * h2 * w2) {
        const int b = (int)(orow / (h2 * w2));
        const int rem = (int)(orow - (int64_t)b * h2 * w2);
        const int y2 = rem / w2, x2 = rem - y2 * w2;
        for (int dy = 0; dy < ps; ++dy)
            for (int dx = 0; dx < ps; ++dx) {
                int64_t tok = tokens[((int64_t)b * H + y2 * ps + dy) * W + x2 * ps + dx];
                tok = tok < 0 ? 0 : (tok >= num_labels ? num_labels - 1 : tok);
                const float* e = emb + tok * c_in;
                float s = 0.f;
                for (int c = lane; c < c_in; c += 32) s += e[c];
                const float mean = warp_sum(s) / c_in;
                float v = 0.f;
                for (int c = lane; c < c_in; c += 32) { const float d = e[c] - mean; v = fmaf(d, d, v); }
                const float rstd = ln_rstd(warp_sum(v) / c_in);
                for (int c = lane; c < c_in; c += 32) srow[c * ps * ps + dy * ps + dx] = __float2half_rn((e[c] - mean) * rstd);
            }
    }
    __syncwarp();
    if (orow < (int64_t)B * h2 * w2) {
        __half* o = out + orow * rowlen;
        if ((rowlen & 7) == 0) {
            for (int i = lane * 8; i < rowlen; i += 256) *reinterpret_cast<uint4*>(o + i) = *reinterpret_cast<const uint4*>(srow + i);
        } else {
            for (int i = lane; i < rowlen; i += 32) o[i] = srow[i];
        }
    }
}

int launch_embed_tokens(const int64_t* tokens, const float* emb, int num_labels, int c_in, int B, int H, int W, int ps,
                        __half* out, cudaStream_t st) {
    ProfScope prof("embed_tokens", (double)B * H * W * c_in * 6.0, st);
    PB_CHECK(H % ps == 0 && W % ps == 0, "embed: latent %dx%d not divisible by patch_size %d", H, W, ps);
    const int64_t rows = (int64_t)B * (H / ps) * (W / ps);
    const size_t smem = (size_t)8 * c_in * ps * ps * sizeof(__half);
    PB_CHECK(smem <= 48 * 1024, "embed: c_in*patch^2 too large");
    embed_tokens_kernel<<<ceil_div(rows, 8), 256, smem, st>>>(tokens, emb, num_labels, c_in, B, H, W, ps, out);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ LayerNorm over rows (warp per row)
template <bool PATCHIFY>
__global__ void __launch_bounds__(256) ln_rows_kernel(const float* __restrict__ x, int64_t rows, int C, float scale,
                                                      float shift, __half* __restrict__ out16, float* __restrict__ out32,
                                                      int h, int w, float* __restrict__ mean_out) {
    pdl_launch_dependents();
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + row * C);
    const int nv = C >> 2;
    float s = 0.f;
    for (int i = lane; i < nv; i += 32) { const float4 v = xr[i]; s += (v.x + v.y) + (v.z + v.w); }
    const float mean = warp_sum(s) / C;
    if (mean_out && lane == 0) mean_out[row] = mean;
    float q = 0.f;
    for (int i = lane; i < nv; i += 32) {
        const float4 v = xr[i];
        const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = ln_rstd(warp_sum(q) / C) * scale;
    int64_t obase = row * C;
    if (PATCHIFY) {   // row = (b, y, x) on an h x w grid -> out row (b, y/2, x/2), column block (y%2*2 + x%2)
        const int64_t hw = (int64_t)h * w;
        const int64_t b = row / hw;
        const int rem = (int)(row - b * hw);
        const int y = rem / w, xx = rem - y * w;
        obase = ((b * (h >> 1) + (y >> 1)) * (w >> 1) + (xx >> 1)) * (4 * (int64_t)C) + ((y & 1) * 2 + (xx & 1)) * C;
    }
    for (int i = lane; i < nv; i += 32) {
        const float4 v = xr[i];
        const float a = fmaf(v.x - mean, rstd, shift), b = fmaf(v.y - mean, rstd, shift);
        const float c = fmaf(v.z - mean, rstd, shift), d = fmaf(v.w - mean, rstd, shift);
        if (out16) {
            uint2 pk;
            pk.x = pack_half2(a, b);
            pk.y = pack_half2(c, d);
            *reinterpret_cast<uint2*>(out16 + obase + i * 4) = pk;
        } else {
            *reinterpret_cast<float4*>(out32 + obase + i * 4) = make_float4(a, b, c, d);
        }
    }
}

int launch_ln_rows(const float* x, int64_t rows, int C, float scale, float shift, __half* out16, float* out32,
                   cudaStream_t st, float* mean_out) {
    ProfScope prof("layernorm", (double)rows * C * (out16 ? 6.0 : 8.0), st);
    PB_CHECK(C % 4 == 0, "layernorm: C=%d must be a multiple of 4", C);
    PB_CHECK((out16 != nullptr) != (out32 != nullptr), "layernorm: exactly one output");
    if (rows == 0) return 0;
    ln_rows_kernel<false><<<ceil_div(rows, 8), 256, 0, st>>>(x, rows, C, scale, shift, out16, out32, 0, 0, mean_out);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_ln_patchify2(const float* x, int B, int h, int w, int c, __half* out, cudaStream_t st) {
    ProfScope prof("layernorm", (double)B * h * w * c * 6.0, st);
    PB_CHECK(c % 4 == 0 && h % 2 == 0 && w % 2 == 0, "ln_patchify: bad geometry %dx%dx%d", h, w, c);
    const int64_t rows = (int64_t)B * h * w;
    ln_rows_kernel<true><<<ceil_div(rows, 8), 256, 0, st>>>(x, rows, c, 1.0f, 0.0f, out, nullptr, h, w, nullptr);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ depthwise conv + LayerNorm (warp per position)
// NV = float4 chunks per lane: supports c <= NV*128.
// WRAP: per-sample seamless tiling.  Sample b reads the byte wrap[b < n_base ? b : b - n_base] (the unconditional rows of a
// CFG batch, b >= n_base, read the byte of their pair); bit 0 wraps x, bit 1 wraps y.  On a wrapped axis every tap reads its
// coordinate modulo the grid size (Conv2d padding_mode='circular', also on grids smaller than the kernel); on an unwrapped
// axis the arithmetic is the zero-padding instance's, so a byte-0 sample gives its bits.
__device__ __forceinline__ int wrap_mod(int i, int n) { const int r = i % n; return r < 0 ? r + n : r; }

__device__ __forceinline__ int wrap_code(const uint8_t* __restrict__ wrap, int b, int n_base) {
    return wrap[b < n_base ? b : b - n_base];
}

template <int NV, bool SKIP, bool WRAP>
__global__ void __launch_bounds__(128) dwconv_ln_kernel(const float* __restrict__ x, const float* __restrict__ skip,
                                                        const float* __restrict__ wp, const float* __restrict__ bias,
                                                        int B, int h, int w, int c, int k, __half* __restrict__ out,
                                                        const uint8_t* __restrict__ wrap, int n_base) {
    // one CTA = a 2x2 patch of positions of one sample (4 warps, small CTAs for occupancy); the four 3x3 halos overlap so
    // half of the tap rows come from L1
    pdl_launch_dependents();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int pw = (w + 1) >> 1, ph = (h + 1) >> 1;
    const int b = blockIdx.x / (pw * ph);
    const int pr = blockIdx.x - b * (pw * ph);
    const int y = (pr / pw) * 2 + (wid >> 1), xx = (pr % pw) * 2 + (wid & 1);
    if (y >= h || xx >= w) return;
    const int64_t pos = ((int64_t)b * h + y) * w + xx;
    const int nvq = c >> 2;          // float4 chunks in a row
    const int pad = k >> 1;
    const int wc = WRAP ? wrap_code(wrap, b, n_base) : 0;
    float4 acc[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int q = i * 32 + lane;
        acc[i] = q < nvq ? __ldg(reinterpret_cast<const float4*>(bias) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int ky = 0; ky < k; ++ky) {
        int iy = y + ky - pad;
        if (WRAP && (wc & 2)) iy = wrap_mod(iy, h);
        else if (iy < 0 || iy >= h) continue;
        for (int kx = 0; kx < k; ++kx) {
            int ix = xx + kx - pad;
            if (WRAP && (wc & 1)) ix = wrap_mod(ix, w);
            else if (ix < 0 || ix >= w) continue;
            const int64_t ipos = ((int64_t)b * h + iy) * w + ix;
            const int tap = ky * k + kx;
            if (!SKIP) {
                const float4* xr = reinterpret_cast<const float4*>(x + ipos * c);
                const float4* wr = reinterpret_cast<const float4*>(wp + (int64_t)tap * c);
#pragma unroll
                for (int i = 0; i < NV; ++i) {
                    const int q = i * 32 + lane;
                    if (q < nvq) {
                        const float4 v = xr[q], ww = __ldg(wr + q);
                        acc[i].x = fmaf(v.x, ww.x, acc[i].x); acc[i].y = fmaf(v.y, ww.y, acc[i].y);
                        acc[i].z = fmaf(v.z, ww.z, acc[i].z); acc[i].w = fmaf(v.w, ww.w, acc[i].w);
                    }
                }
            } else {
                // output channels g = 4q..4q+3 read concatenated [x, skip] channels 8q..8q+7
                const float4* w0 = reinterpret_cast<const float4*>(wp + ((int64_t)tap * 2 + 0) * c);
                const float4* w1 = reinterpret_cast<const float4*>(wp + ((int64_t)tap * 2 + 1) * c);
#pragma unroll
                for (int i = 0; i < NV; ++i) {
                    const int q = i * 32 + lane;
                    if (q < nvq) {
                        const int cc = 8 * q;
                        const float* src = cc < c ? x + ipos * c + cc : skip + ipos * c + (cc - c);
                        const float4 lo = *reinterpret_cast<const float4*>(src);
                        const float4 hi = *reinterpret_cast<const float4*>(src + 4);
                        const float4 a = __ldg(w0 + q), bb = __ldg(w1 + q);
                        acc[i].x = fmaf(lo.x, a.x, fmaf(lo.y, bb.x, acc[i].x));
                        acc[i].y = fmaf(lo.z, a.y, fmaf(lo.w, bb.y, acc[i].y));
                        acc[i].z = fmaf(hi.x, a.z, fmaf(hi.y, bb.z, acc[i].z));
                        acc[i].w = fmaf(hi.z, a.w, fmaf(hi.w, bb.w, acc[i].w));
                    }
                }
            }
        }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
        if (i * 32 + lane < nvq) s += (acc[i].x + acc[i].y) + (acc[i].z + acc[i].w);
    const float mean = warp_sum(s) / c;
    float qv = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
        if (i * 32 + lane < nvq) {
            const float a = acc[i].x - mean, bq = acc[i].y - mean, cq = acc[i].z - mean, d = acc[i].w - mean;
            qv += (a * a + bq * bq) + (cq * cq + d * d);
        }
    const float rstd = ln_rstd(warp_sum(qv) / c);
    __half* o = out + pos * c;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
        const int q = i * 32 + lane;
        if (q < nvq) {
            uint2 pk;
            pk.x = pack_half2((acc[i].x - mean) * rstd, (acc[i].y - mean) * rstd);
            pk.y = pack_half2((acc[i].z - mean) * rstd, (acc[i].w - mean) * rstd);
            *reinterpret_cast<uint2*>(o + q * 4) = pk;
        }
    }
}

// ------------------------------------------------------------------ depthwise 3x3 conv + LayerNorm (thread per 4 channels)
// The warp-per-position kernel above issues 9 activation + 9 weight loads per position and float4 chunk and is bound
// by LSU/L1 issue, not by HBM.  Here a thread owns 4 output channels of a
// 2-row x 8-column patch of positions: it walks the patch's 4 x 10 input halo once (2.5 loads per output instead of
// 18), keeps the 16 accumulators in registers, and the CTA (c/4 threads) then reduces the LayerNorm statistics of
// its 16 positions through shared memory.  Tap order per output is (ky, kx) ascending, as in the kernel above.
constexpr int DW_PH = 2, DW_PW = 8, DW_NPOS = DW_PH * DW_PW;

__device__ __forceinline__ void fma4(float4& a, const float4& v, const float4& w) {
    a.x = fmaf(v.x, w.x, a.x); a.y = fmaf(v.y, w.y, a.y); a.z = fmaf(v.z, w.z, a.z); a.w = fmaf(v.w, w.w, a.w);
}

// sum of s[p] over the CTA's threads for p < 16; result in tot[p] (shared; two __syncthreads)
__device__ __forceinline__ void block_sum16(float (&s)[DW_NPOS], float* red, float* tot, int n_warps) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    // transpose-reduce: after the o = 8,4,2,1 steps lane l holds position (l & 15) summed over its 16-lane half
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
#pragma unroll
        for (int i = 0; i < o; ++i) {
            const bool up = (lane & o) != 0;
            const float send = up ? s[i] : s[i + o];
            const float keep = up ? s[i + o] : s[i];
            s[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
    s[0] += __shfl_xor_sync(0xffffffffu, s[0], 16);
    // lane l < 16 now holds position bitrev-free index: bit o of the lane selected the upper half at step o -> p = l & 15
    if (lane < DW_NPOS) red[wid * DW_NPOS + lane] = s[0];
    __syncthreads();
    if (threadIdx.x < DW_NPOS) {
        float t = 0.f;
        for (int i = 0; i < n_warps; ++i) t += red[i * DW_NPOS + threadIdx.x];
        tot[threadIdx.x] = t;
    }
    __syncthreads();
}

// WRAP: as in dwconv_ln_kernel.  An unwrapped y keeps the CTA-uniform row test; a wrapped axis reads its halo modulo the grid.
template <bool SKIP, int MAXT, bool WRAP>
__global__ void __launch_bounds__(MAXT, (MAXT == 320 ? 2 : 1)) dwconv3_ln_patch_kernel(const float* __restrict__ x, const float* __restrict__ skip,
                                                                const float* __restrict__ wp, const float* __restrict__ bias,
                                                                int B, int h, int w, int c, __half* __restrict__ out,
                                                                const uint8_t* __restrict__ wrap, int n_base) {
    __shared__ float red[32 * DW_NPOS];
    __shared__ float tot[2][DW_NPOS];
    pdl_launch_dependents();
    const int q = threadIdx.x, nvq = c >> 2;
    const bool active = q < nvq;
    const int qc = active ? q : 0;                       // idle threads shadow chunk 0 and never store
    const int tiles_x = (w + DW_PW - 1) / DW_PW, tiles_y = (h + DW_PH - 1) / DW_PH;
    const int b = blockIdx.x / (tiles_x * tiles_y);
    const int tr = blockIdx.x - b * (tiles_x * tiles_y);
    const int y0 = (tr / tiles_x) * DW_PH, x0 = (tr % tiles_x) * DW_PW;
    const int wc = WRAP ? wrap_code(wrap, b, n_base) : 0;

    float4 acc[DW_PH][DW_PW];
    {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias) + qc);
#pragma unroll
        for (int oy = 0; oy < DW_PH; ++oy)
#pragma unroll
            for (int ox = 0; ox < DW_PW; ++ox) acc[oy][ox] = bv;
    }
#pragma unroll
    for (int r = 0; r < DW_PH + 2; ++r) {
        int iy = y0 - 1 + r;
        if (WRAP && (wc & 2)) iy = wrap_mod(iy, h);
        else if (iy < 0 || iy >= h) continue;            // CTA-uniform: a zero-padding row contributes nothing
        // input row r feeds output row oy with ky = r - oy
        float4 wt[DW_PH][3][SKIP ? 2 : 1];
#pragma unroll
        for (int oy = 0; oy < DW_PH; ++oy) {
            const int ky = r - oy;
            if (ky < 0 || ky > 2) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int tap = ky * 3 + kx;
                if (SKIP) {
                    wt[oy][kx][0] = __ldg(reinterpret_cast<const float4*>(wp + ((int64_t)tap * 2 + 0) * c) + qc);
                    wt[oy][kx][SKIP ? 1 : 0] = __ldg(reinterpret_cast<const float4*>(wp + ((int64_t)tap * 2 + 1) * c) + qc);
                } else {
                    wt[oy][kx][0] = __ldg(reinterpret_cast<const float4*>(wp + (int64_t)tap * c) + qc);
                }
            }
        }
        const int64_t rowbase = ((int64_t)b * h + iy) * w;
#pragma unroll
        for (int j = 0; j < DW_PW + 2; ++j) {
            int ix = x0 - 1 + j;
            if (WRAP && (wc & 1)) ix = wrap_mod(ix, w);
            const bool ok = ix >= 0 && ix < w;
            const int64_t ipos = rowbase + (ok ? ix : x0);
            float4 v0, v1;
            if (SKIP) {
                // output channels 4q..4q+3 read concatenated [x, skip] channels 8q..8q+7
                const int cc = 8 * qc;
                const float* src = cc < c ? x + ipos * c + cc : skip + ipos * c + (cc - c);
                v0 = *reinterpret_cast<const float4*>(src);
                v1 = *reinterpret_cast<const float4*>(src + 4);
            } else {
                v0 = *(reinterpret_cast<const float4*>(x + ipos * c) + qc);
                v1 = v0;
            }
            if (!ok) { v0 = make_float4(0.f, 0.f, 0.f, 0.f); v1 = v0; }
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ox = j - kx;
                if (ox < 0 || ox >= DW_PW) continue;
#pragma unroll
                for (int oy = 0; oy < DW_PH; ++oy) {
                    const int ky = r - oy;
                    if (ky < 0 || ky > 2) continue;
                    float4& a = acc[oy][ox];
                    if (SKIP) {
                        const float4 wa = wt[oy][kx][0], wb = wt[oy][kx][SKIP ? 1 : 0];
                        a.x = fmaf(v0.x, wa.x, fmaf(v0.y, wb.x, a.x));
                        a.y = fmaf(v0.z, wa.y, fmaf(v0.w, wb.y, a.y));
                        a.z = fmaf(v1.x, wa.z, fmaf(v1.y, wb.z, a.z));
                        a.w = fmaf(v1.z, wa.w, fmaf(v1.w, wb.w, a.w));
                    } else {
                        fma4(a, v0, wt[oy][kx][0]);
                    }
                }
            }
        }
    }
    // ---- LayerNorm over channels for the 16 positions (two-pass, like F.layer_norm)
    const int n_warps = blockDim.x >> 5;
    float s[DW_NPOS];
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const float4 a = acc[p / DW_PW][p % DW_PW];
        s[p] = active ? (a.x + a.y) + (a.z + a.w) : 0.f;
    }
    block_sum16(s, red, tot[0], n_warps);
    const float inv_c = 1.0f / c;
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const float mean = tot[0][p] * inv_c;
        const float4 a = acc[p / DW_PW][p % DW_PW];
        const float d0 = a.x - mean, d1 = a.y - mean, d2 = a.z - mean, d3 = a.w - mean;
        s[p] = active ? (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3) : 0.f;
    }
    block_sum16(s, red, tot[1], n_warps);
    if (!active) return;
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const int y = y0 + p / DW_PW, xx = x0 + p % DW_PW;
        if (y >= h || xx >= w) continue;
        const float mean = tot[0][p] * inv_c;
        const float rstd = ln_rstd(tot[1][p] * inv_c);
        const float4 a = acc[p / DW_PW][p % DW_PW];
        uint2 pk;
        pk.x = pack_half2((a.x - mean) * rstd, (a.y - mean) * rstd);
        pk.y = pack_half2((a.z - mean) * rstd, (a.w - mean) * rstd);
        *reinterpret_cast<uint2*>(out + (((int64_t)b * h + y) * w + xx) * c + q * 4) = pk;
    }
}

static int dwconv3_patch_launch(const float* x, const float* skip, const float* wp, const float* bias, int B, int h, int w,
                                int c, __half* out, const uint8_t* wrap, int n_base, cudaStream_t st) {
    const int64_t grid = (int64_t)B * ceil_div(h, DW_PH) * ceil_div(w, DW_PW);
    PB_CHECK(grid < (1ll << 31), "dwconv: grid too large");
    const int threads = ceil_div(c / 4, 32) * 32;
#define PB_DW_LAUNCH_W(MAXT, WRAP)                                                                                      \
    do {                                                                                                                \
        if (skip)                                                                                                       \
            dwconv3_ln_patch_kernel<true, MAXT, WRAP><<<(unsigned)grid, threads, 0, st>>>(x, skip, wp, bias, B, h, w, c, out, \
                                                                                          wrap, n_base);                \
        else                                                                                                            \
            dwconv3_ln_patch_kernel<false, MAXT, WRAP><<<(unsigned)grid, threads, 0, st>>>(x, skip, wp, bias, B, h, w, c, out, \
                                                                                           wrap, n_base);               \
    } while (0)
#define PB_DW_LAUNCH(MAXT)                   \
    do {                                     \
        if (wrap) PB_DW_LAUNCH_W(MAXT, true); \
        else PB_DW_LAUNCH_W(MAXT, false);     \
    } while (0)
    if (threads <= 64) PB_DW_LAUNCH(64);
    else if (threads <= 160) PB_DW_LAUNCH(160);
    else if (threads <= 320) PB_DW_LAUNCH(320);
    else PB_DW_LAUNCH(640);
#undef PB_DW_LAUNCH
#undef PB_DW_LAUNCH_W
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ codec ResBlock front, fused (ref/src/vqgan.py:36-40)
//   x' = x + g2 * (dw3x3(ReplicationPad(LN(x) * (1 + g0) + g1)) + bias);   a16 = fp16(LN(x') * (1 + g3) + g4)
// Three launches (LayerNorm -> fp32 copy, depthwise + residual, LayerNorm -> fp16) moved 26 bytes per element; here a warp-per-row
// statistics pre-pass (mean, rstd of every position: 4 B read per element) feeds ONE patch kernel that normalises the halo values
// on the fly (LayerNorm is affine per position), keeps the 2 x 8 patch in registers, adds the residual and reduces the second
// LayerNorm's statistics inside the CTA (thread = 4 channels, like dwconv3_ln_patch_kernel): 4 + 4 + 4 + 2 = 14 bytes per element.
// x' goes to a SECOND buffer (neighbouring CTAs still read the old x for their halos); the MLP's second GEMM reads it as the
// residual and writes the block's output back into the original buffer.
__global__ void __launch_bounds__(256) row_stats_kernel(const float* __restrict__ x, int64_t rows, int C, float2* __restrict__ stats) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float4* xr = reinterpret_cast<const float4*>(x + row * C);
    const int nv = C >> 2;
    float s = 0.f;
    for (int i = lane; i < nv; i += 32) { const float4 v = xr[i]; s += (v.x + v.y) + (v.z + v.w); }
    const float mean = warp_sum(s) / C;
    float q = 0.f;
    for (int i = lane; i < nv; i += 32) {
        const float4 v = xr[i];
        const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = ln_rstd(warp_sum(q) / C);
    if (lane == 0) stats[row] = make_float2(mean, rstd);
}

// WRAP: per-sample seamless tiling (wrap[b], bit 0 = x, bit 1 = y): a wrapped axis replaces ReplicationPad2d's clamped coordinate
// by the coordinate modulo the grid size (circular padding); an unwrapped one keeps the clamp.
template <int MAXT, int MINB, bool WRAP>
__global__ void __launch_bounds__(MAXT, MINB) vq_front_patch_kernel(const float* __restrict__ x, const float2* __restrict__ stats,
                                                              const float* __restrict__ wp, const float* __restrict__ bias,
                                                              float a0, float g1, float g2, float a3, float g4, int B, int h, int w,
                                                              int c, float* __restrict__ x_out, __half* __restrict__ a16,
                                                              const uint8_t* __restrict__ wrap) {
    __shared__ float red[32 * DW_NPOS];
    __shared__ float tot[2][DW_NPOS];
    __shared__ float2 st_s[DW_PH + 2][DW_PW + 2];
    const int q = threadIdx.x, nvq = c >> 2;
    const bool active = q < nvq;
    const int qc = active ? q : 0;                       // idle threads shadow chunk 0 and never store
    const int tiles_x = (w + DW_PW - 1) / DW_PW, tiles_y = (h + DW_PH - 1) / DW_PH;
    const int b = blockIdx.x / (tiles_x * tiles_y);
    const int tr = blockIdx.x - b * (tiles_x * tiles_y);
    const int y0 = (tr / tiles_x) * DW_PH, x0 = (tr % tiles_x) * DW_PW;
    const int wc = WRAP ? wrap[b] : 0;
    // ReplicationPad2d(1) = clamped coordinates; circular on a wrapped axis
    auto cy = [&](int y) { return (WRAP && (wc & 2)) ? wrap_mod(y, h) : min(max(y, 0), h - 1); };
    auto cx = [&](int xx) { return (WRAP && (wc & 1)) ? wrap_mod(xx, w) : min(max(xx, 0), w - 1); };
    if (threadIdx.x < (DW_PH + 2) * (DW_PW + 2)) {
        const int r = threadIdx.x / (DW_PW + 2), j = threadIdx.x - r * (DW_PW + 2);
        st_s[r][j] = stats[((int64_t)b * h + cy(y0 - 1 + r)) * w + cx(x0 - 1 + j)];
    }
    __syncthreads();

    float4 acc[DW_PH][DW_PW];
    {
        const float4 bv = __ldg(reinterpret_cast<const float4*>(bias) + qc);
#pragma unroll
        for (int oy = 0; oy < DW_PH; ++oy)
#pragma unroll
            for (int ox = 0; ox < DW_PW; ++ox) acc[oy][ox] = bv;
    }
#pragma unroll
    for (int r = 0; r < DW_PH + 2; ++r) {
        float4 wt[DW_PH][3];
#pragma unroll
        for (int oy = 0; oy < DW_PH; ++oy) {
            const int ky = r - oy;
            if (ky < 0 || ky > 2) continue;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) wt[oy][kx] = __ldg(reinterpret_cast<const float4*>(wp + (int64_t)(ky * 3 + kx) * c) + qc);
        }
        const int64_t rowbase = ((int64_t)b * h + cy(y0 - 1 + r)) * w;
#pragma unroll
        for (int j = 0; j < DW_PW + 2; ++j) {
            const float4 v = *(reinterpret_cast<const float4*>(x + (rowbase + cx(x0 - 1 + j)) * c) + qc);
            const float2 ms = st_s[r][j];
            const float sc = ms.y * a0;                   // the first LayerNorm's scalar affine, as launch_ln_rows applies it
            const float4 t = make_float4(fmaf(v.x - ms.x, sc, g1), fmaf(v.y - ms.x, sc, g1), fmaf(v.z - ms.x, sc, g1), fmaf(v.w - ms.x, sc, g1));
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int ox = j - kx;
                if (ox < 0 || ox >= DW_PW) continue;
#pragma unroll
                for (int oy = 0; oy < DW_PH; ++oy) {
                    const int ky = r - oy;
                    if (ky < 0 || ky > 2) continue;
                    fma4(acc[oy][ox], t, wt[oy][kx]);
                }
            }
        }
    }
    // ---- residual: x' = x + g2 * conv (the centre values come back from L1)
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const float4 xc = *(reinterpret_cast<const float4*>(x + (((int64_t)b * h + cy(y0 + p / DW_PW)) * w + cx(x0 + p % DW_PW)) * c) + qc);
        float4& a = acc[p / DW_PW][p % DW_PW];
        a.x = fmaf(a.x, g2, xc.x); a.y = fmaf(a.y, g2, xc.y); a.z = fmaf(a.z, g2, xc.z); a.w = fmaf(a.w, g2, xc.w);
    }
    // ---- second LayerNorm over channels for the 16 positions (two-pass, like F.layer_norm)
    const int n_warps = blockDim.x >> 5;
    float s[DW_NPOS];
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const float4 a = acc[p / DW_PW][p % DW_PW];
        s[p] = active ? (a.x + a.y) + (a.z + a.w) : 0.f;
    }
    block_sum16(s, red, tot[0], n_warps);
    const float inv_c = 1.0f / c;
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const float mean = tot[0][p] * inv_c;
        const float4 a = acc[p / DW_PW][p % DW_PW];
        const float d0 = a.x - mean, d1 = a.y - mean, d2 = a.z - mean, d3 = a.w - mean;
        s[p] = active ? (d0 * d0 + d1 * d1) + (d2 * d2 + d3 * d3) : 0.f;
    }
    block_sum16(s, red, tot[1], n_warps);
    if (!active) return;
#pragma unroll
    for (int p = 0; p < DW_NPOS; ++p) {
        const int y = y0 + p / DW_PW, xx = x0 + p % DW_PW;
        if (y >= h || xx >= w) continue;
        const float mean = tot[0][p] * inv_c;
        const float rstd = ln_rstd(tot[1][p] * inv_c) * a3;
        const float4 a = acc[p / DW_PW][p % DW_PW];
        const int64_t o = (((int64_t)b * h + y) * w + xx) * c + q * 4;
        *reinterpret_cast<float4*>(x_out + o) = a;
        uint2 pk;
        pk.x = pack_half2(fmaf(a.x - mean, rstd, g4), fmaf(a.y - mean, rstd, g4));
        pk.y = pack_half2(fmaf(a.z - mean, rstd, g4), fmaf(a.w - mean, rstd, g4));
        *reinterpret_cast<uint2*>(a16 + o) = pk;
    }
}

bool vq_front_fused_ok(int c, int h, int w) { return c % 4 == 0 && c >= 4 * (DW_PH + 2) * (DW_PW + 2) && c <= 512 && h >= 1 && w >= 1; }

int launch_vq_front_fused(const float* x, int B, int h, int w, int c, const float* w9, const float* bias, const float* gam,
                          float2* stats_scratch, float* x_out, __half* a16, cudaStream_t st, const uint8_t* wrap) {
    PB_CHECK(vq_front_fused_ok(c, h, w), "vq_front: width %d not handled by the patch kernel", c);
    const int64_t M = (int64_t)B * h * w;
    if (M == 0) return 0;
    {
        ProfScope prof("vq_rowstats", (double)M * c * 4.0, st);
        row_stats_kernel<<<ceil_div(M, 8), 256, 0, st>>>(x, M, c, stats_scratch);
        PB_LAUNCH_CHECK();
    }
    ProfScope prof("vq_front", (double)M * c * 10.0, st);
    const int64_t grid = (int64_t)B * ceil_div(h, DW_PH) * ceil_div(w, DW_PW);
    PB_CHECK(grid < (1ll << 31), "vq_front: grid too large");
    const int threads = ceil_div(c / 4, 32) * 32;
    // 3 CTAs of 96 threads per SM at 168 registers (capping at 128 registers for a fourth CTA spills)
#define PB_VQF_LAUNCH(MAXT, MINB, WRAP)                                                                                 \
    vq_front_patch_kernel<MAXT, MINB, WRAP><<<(unsigned)grid, threads, 0, st>>>(x, stats_scratch, w9, bias, 1.0f + gam[0], gam[1], \
                                                                                gam[2], 1.0f + gam[3], gam[4], B, h, w, c, x_out,  \
                                                                                a16, wrap)
    if (threads <= 64) {
        if (wrap) PB_VQF_LAUNCH(64, 6, true);
        else PB_VQF_LAUNCH(64, 6, false);
    } else {
        if (wrap) PB_VQF_LAUNCH(128, 3, true);
        else PB_VQF_LAUNCH(128, 3, false);
    }
#undef PB_VQF_LAUNCH
    PB_LAUNCH_CHECK();
    return 0;
}

template <int NV>
static int dwconv_dispatch(const float* x, const float* skip, const float* wp, const float* bias, int B, int h, int w,
                           int c, int k, __half* out, const uint8_t* wrap, int n_base, cudaStream_t st) {
    const int64_t grid = (int64_t)B * ((h + 1) / 2) * ((w + 1) / 2);
    PB_CHECK(grid < (1ll << 31), "dwconv: grid too large");
    if (skip && wrap)
        dwconv_ln_kernel<NV, true, true><<<(unsigned)grid, 128, 0, st>>>(x, skip, wp, bias, B, h, w, c, k, out, wrap, n_base);
    else if (wrap)
        dwconv_ln_kernel<NV, false, true><<<(unsigned)grid, 128, 0, st>>>(x, skip, wp, bias, B, h, w, c, k, out, wrap, n_base);
    else if (skip)
        dwconv_ln_kernel<NV, true, false><<<(unsigned)grid, 128, 0, st>>>(x, skip, wp, bias, B, h, w, c, k, out, wrap, n_base);
    else
        dwconv_ln_kernel<NV, false, false><<<(unsigned)grid, 128, 0, st>>>(x, skip, wp, bias, B, h, w, c, k, out, wrap, n_base);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_dwconv_ln(const float* x, const float* skip, const float* w_packed, const float* bias, int B, int h, int w,
                     int c, int k, __half* out, cudaStream_t st, const uint8_t* wrap, int n_base) {
    ProfScope prof("dwconv_ln", (double)B * h * w * c * (skip ? 10.0 : 6.0), st);
    PB_CHECK(c % 8 == 0, "dwconv: c=%d must be a multiple of 8", c);
    PB_CHECK(k % 2 == 1, "dwconv: kernel_size %d must be odd", k);
    static const bool old_kernel = getenv("PB200_DWCONV_WARP") != nullptr;      // A/B knob
    // the patch kernel takes the wide levels only: at 640 channels its 152 registers x 160 threads leave 15% occupancy
    static const bool patch_all = getenv("PB200_DWCONV_PATCH") != nullptr;
    if (k == 3 && c <= 2560 && !old_kernel && (patch_all || (c > 640 && w >= DW_PW)))
        return dwconv3_patch_launch(x, skip, w_packed, bias, B, h, w, c, out, wrap, n_base, st);
    if (c <= 128) return dwconv_dispatch<1>(x, skip, w_packed, bias, B, h, w, c, k, out, wrap, n_base, st);
    if (c <= 640) return dwconv_dispatch<5>(x, skip, w_packed, bias, B, h, w, c, k, out, wrap, n_base, st);
    if (c <= 1280) return dwconv_dispatch<10>(x, skip, w_packed, bias, B, h, w, c, k, out, wrap, n_base, st);
    if (c <= 2560) return dwconv_dispatch<20>(x, skip, w_packed, bias, B, h, w, c, k, out, wrap, n_base, st);
    PB_CHECK(false, "dwconv: c=%d > 2560 unsupported", c);
    return 1;
}

// ------------------------------------------------------------------ GlobalResponseNorm
// Two launches: (1) grn_scale_kernel, one CTA per sample: the normaliser mean_n sqrt(sq[b,n]) and the per-(sample, channel)
// multiplier 1 + gamma[n] * Gx / (mean Gx + 1e-6) -> fp32 scale[b, n]; it also zeroes sq_next (the other half of the
// ping-pong pair) for the next block's GEMM epilogue, so the statistic being read is never written in the same launch.
// (2) grn_apply_kernel: a pure streaming pass h = h * scale[b, n] + beta[n] over the fp16 hidden with no per-CTA prologue
// (the round-1 single kernel recomputed the N-term normaliser in EVERY CTA before its first load: 3.0 TB/s at 27 %
// occupancy in ncu; the stream itself is now the only thing a CTA does).
__device__ __forceinline__ float grn_fx(unsigned long long q) { return __ull2float_rn(q) * (1.0f / 16777216.0f); }

__global__ void __launch_bounds__(512) grn_scale_kernel(int N, const unsigned long long* __restrict__ sq,
                                                        unsigned long long* __restrict__ sq_next, const float* __restrict__ gamma,
                                                        float* __restrict__ scale, int zero_per_sample) {
    pdl_launch_dependents();
    const int b = blockIdx.x;
    const unsigned long long* sqb = sq + (int64_t)b * N;
    float s = 0.f;
    for (int i = threadIdx.x; i < (N >> 1); i += blockDim.x) {
        const ulonglong2 q = *reinterpret_cast<const ulonglong2*>(sqb + 2 * i);
        s += sqrtf(grn_fx(q.x)) + sqrtf(grn_fx(q.y));
    }
    __shared__ float red[16];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    float tot = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
    const float inv_denom = 1.0f / (tot / N + 1e-6f);
    for (int i = threadIdx.x; i < N; i += blockDim.x)
        scale[(int64_t)b * N + i] = fmaf(__ldg(gamma + i), sqrtf(grn_fx(sqb[i])) * inv_denom, 1.0f);
    for (int i = threadIdx.x; i < zero_per_sample; i += blockDim.x) sq_next[(int64_t)b * zero_per_sample + i] = 0ull;
}

// grid (column groups of 8 channels x GRN_TPB threads, row groups, samples); each thread owns 8 channels and walks
// rows_per_cta rows with 8 independent 16-byte loads in flight
constexpr int GRN_ROWS = 8;
__global__ void __launch_bounds__(256) grn_apply_kernel(__half* __restrict__ h, int P, int N, const float* __restrict__ scale,
                                                        const float* __restrict__ beta, int rows_per_cta) {
    pdl_launch_dependents();
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= (N >> 3)) return;
    const int b = blockIdx.z, col = ch * 8;
    const int r0 = blockIdx.y * rows_per_cta, r1 = min(P, r0 + rows_per_cta);
    __half* hb = h + ((int64_t)b * P) * N + col;
    // issue the first row group's loads before the (L2-resident) scale / beta vectors are needed
    uint4 v[GRN_ROWS];
#pragma unroll
    for (int u = 0; u < GRN_ROWS; ++u)
        if (r0 + u < r1) v[u] = *reinterpret_cast<const uint4*>(hb + (int64_t)(r0 + u) * N);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + (int64_t)b * N + col)), s1 = __ldg(reinterpret_cast<const float4*>(scale + (int64_t)b * N + col + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + col)), b1 = __ldg(reinterpret_cast<const float4*>(beta + col + 4));
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    for (int r = r0; r < r1; r += GRN_ROWS) {
        uint4 nx[GRN_ROWS];
        const int rn = r + GRN_ROWS;
#pragma unroll
        for (int u = 0; u < GRN_ROWS; ++u)
            if (rn + u < r1) nx[u] = *reinterpret_cast<const uint4*>(hb + (int64_t)(rn + u) * N);      // next group in flight
#pragma unroll
        for (int u = 0; u < GRN_ROWS; ++u) {
            if (r + u < r1) {
                __half2* hv = reinterpret_cast<__half2*>(&v[u]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(hv[j]);
                    hv[j] = __floats2half2_rn(fmaf(f.x, sc[2 * j], be[2 * j]), fmaf(f.y, sc[2 * j + 1], be[2 * j + 1]));
                }
                *reinterpret_cast<uint4*>(hb + (int64_t)(r + u) * N) = v[u];
            }
        }
#pragma unroll
        for (int u = 0; u < GRN_ROWS; ++u) v[u] = nx[u];
    }
}

int launch_grn_fused(__half* h, int B, int P, int N, const uint64_t* sq, uint64_t* sq_next, int zero_per_sample, const float* gamma,
                     const float* beta, float* scale_scratch, cudaStream_t st) {
    ProfScope prof("grn", (double)B * P * N * 4.0, st);
    PB_CHECK(N % 8 == 0, "grn: N=%d must be a multiple of 8", N);
    PB_CHECK(scale_scratch != nullptr, "grn: scale scratch [B, N] fp32 required");
    if (B == 0 || P == 0) return 0;
    PB_CHECK(B <= 65535, "grn: batch too large");
    grn_scale_kernel<<<B, 512, 0, st>>>(N, reinterpret_cast<const unsigned long long*>(sq), reinterpret_cast<unsigned long long*>(sq_next),
                                        gamma, scale_scratch, zero_per_sample);
    PB_LAUNCH_CHECK();
    // rows per CTA: 16 (two 8-row groups, the second in flight while the first is converted), 8 when that leaves SMs idle
    const int nch = N >> 3;
    const int tpb = nch >= 256 ? 256 : ((nch + 31) / 32) * 32;
    int rows_per_cta = P >= 16 ? 16 : P;
    if ((int64_t)ceil_div(P, rows_per_cta) * B * ceil_div(nch, tpb) < 4 * sm_count() && rows_per_cta > 8) rows_per_cta = 8;
    dim3 grid(ceil_div(nch, tpb), ceil_div(P, rows_per_cta), B);
    grn_apply_kernel<<<grid, tpb, 0, st>>>(h, P, N, scale_scratch, beta, rows_per_cta);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ timestep embedding + FiLM table
__global__ void r_embed_kernel(const float* __restrict__ r, int B, int c_r, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * c_r) return;
    const int b = i / c_r, j = i - b * c_r;
    const int half = c_r / 2;
    if (j >= 2 * half) { out[i] = 0.f; return; }          // odd c_r: zero pad
    const int f = j < half ? j : j - half;
    const float kneg = (float)(-(log(10000.0) / (double)(half - 1)));
    const float freq = expf(__fmul_rn((float)f, kneg));
    const float ang = __fmul_rn(__fmul_rn(r[b], 10000.0f), freq);
    out[i] = j < half ? sinf(ang) : cosf(ang);
}

int launch_r_embed(const float* r, int B, int c_r, float* out, cudaStream_t st) {
    ProfScope prof("film", (double)B * c_r * 4.0, st);
    PB_CHECK(c_r >= 4, "c_r=%d too small", c_r);
    r_embed_kernel<<<ceil_div((long)B * c_r, 128), 128, 0, st>>>(r, B, c_r, out);
    PB_LAUNCH_CHECK();
    return 0;
}

// thread = one output feature j, its W row in registers; loops over the batch (r_embed staged in shared memory)
template <int CR>
__global__ void __launch_bounds__(128) film_table_kernel(const float* __restrict__ r_embed, int B, const float* __restrict__ W,
                                                         const float* __restrict__ bias, int total, float* __restrict__ out) {
    extern __shared__ float s_r[];           // [bt, CR]
    const int j = blockIdx.x * 128 + threadIdx.x;
    float wr[CR];
    if (j < total) {
#pragma unroll
        for (int i = 0; i < CR; i += 4) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(W + (int64_t)j * CR + i));
            wr[i] = v.x; wr[i + 1] = v.y; wr[i + 2] = v.z; wr[i + 3] = v.w;
        }
    }
    const float bj = j < total ? bias[j] : 0.f;
    for (int b0 = 0; b0 < B; b0 += 64) {
        const int bt = min(64, B - b0);
        __syncthreads();
        for (int i = threadIdx.x; i < bt * CR; i += 128) s_r[i] = r_embed[(int64_t)b0 * CR + i];
        __syncthreads();
        if (j < total) {
            for (int b = 0; b < bt; ++b) {
                float acc = bj;
#pragma unroll
                for (int i = 0; i < CR; ++i) acc = fmaf(s_r[b * CR + i], wr[i], acc);
                out[(int64_t)(b0 + b) * total + j] = acc;
            }
        }
    }
}

__global__ void film_table_generic_kernel(const float* __restrict__ r_embed, int B, int c_r, const float* __restrict__ W,
                                          const float* __restrict__ bias, int total, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)B * total) return;
    const int b = (int)(i / total), j = (int)(i - (int64_t)b * total);
    float acc = bias[j];
    for (int k = 0; k < c_r; ++k) acc = fmaf(r_embed[b * c_r + k], W[(int64_t)j * c_r + k], acc);
    out[i] = acc;
}

int launch_film_table(const float* r_embed, int B, int c_r, const float* W, const float* bias, int total, float* out,
                      cudaStream_t st) {
    ProfScope prof("film", (double)total * (c_r + B) * 4.0, st);
    if (total == 0) return 0;
    if (c_r == 64)
        film_table_kernel<64><<<ceil_div(total, 128), 128, 64 * 64 * sizeof(float), st>>>(r_embed, B, W, bias, total, out);
    else
        film_table_generic_kernel<<<ceil_div((long)B * total, 256), 256, 0, st>>>(r_embed, B, c_r, W, bias, total, out);
    PB_LAUNCH_CHECK();
    return 0;
}

__global__ void film_apply_kernel(float* __restrict__ x, int64_t M, int N, int P, const float* __restrict__ film,
                                  int64_t film_ld, int64_t film_off) {
    const int nv = N >> 2;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * nv) return;
    const int64_t row = i / nv;
    const int col = (int)(i - row * nv) * 4;
    const float* fa = film + (row / P) * film_ld + film_off + col;
    float4 v = *reinterpret_cast<float4*>(x + row * N + col);
    const float4 a = *reinterpret_cast<const float4*>(fa), s = *reinterpret_cast<const float4*>(fa + N);
    v.x = fmaf(v.x, 1.0f + a.x, s.x); v.y = fmaf(v.y, 1.0f + a.y, s.y);
    v.z = fmaf(v.z, 1.0f + a.z, s.z); v.w = fmaf(v.w, 1.0f + a.w, s.w);
    *reinterpret_cast<float4*>(x + row * N + col) = v;
}

int launch_film_apply(float* x, int64_t M, int N, int P, const float* film, int64_t film_ld, int64_t film_off,
                      cudaStream_t st) {
    ProfScope prof("film", (double)M * N * 8.0, st);
    PB_CHECK(N % 4 == 0 && film_off % 4 == 0 && film_ld % 4 == 0, "film: misaligned table");
    film_apply_kernel<<<ceil_div(M * (N / 4), 256), 256, 0, st>>>(x, M, N, P, film, film_ld, film_off);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ casts
// OP 3: weighted mix with per-row weights: element e takes (wa, wb) = w[3 s], w[3 s + 1] of s = e / per (the sample of its
// row; per = rows per sample * row length), with OP 2's expression.
template <int OP>
__global__ void cast_kernel(const float* __restrict__ a, const float* __restrict__ b, float wa, float wb, int64_t n,
                            __half* __restrict__ out, const float* __restrict__ w = nullptr, int64_t per = 0) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    int64_t s0 = 0;
    if (OP == 3) s0 = i / per;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float t = (i + j < n) ? a[i + j] : 0.f;
        if (OP == 1) t = t / (1.0f + expf(-t));                                   // SiLU
        if (OP == 2) t = b ? fmaf(t, wa, b[(i + j < n) ? i + j : 0] * wb) : t * wa;  // weighted mix
        if (OP == 3) {
            const int64_t s = (i + j >= (s0 + 1) * per) ? s0 + 1 : s0;
            if (i + j < n) t = fmaf(t, w[3 * s], b[i + j] * w[3 * s + 1]);
        }
        v[j] = t;
    }
    if (i + 3 < n && ((reinterpret_cast<uintptr_t>(out + i) & 7) == 0)) {
        uint2 pk;
        pk.x = pack_half2(v[0], v[1]);
        pk.y = pack_half2(v[2], v[3]);
        *reinterpret_cast<uint2*>(out + i) = pk;
    } else {
        for (int j = 0; j < 4 && i + j < n; ++j) out[i + j] = __float2half_rn(v[j]);
    }
}

int launch_cast_f16(const float* x, int64_t n, __half* out, cudaStream_t st) {
    ProfScope prof("cast", (double)n * 6.0, st);
    if (n == 0) return 0;
    cast_kernel<0><<<ceil_div(ceil_div(n, 4), 256), 256, 0, st>>>(x, nullptr, 1.f, 0.f, n, out);
    PB_LAUNCH_CHECK();
    return 0;
}
// fp32 NHWC [B,h,w,c] -> fp16 NHWC [B,h+2,w+2,c] with a border one position wide: sample b's border holds circular copies on
// the axes wrap[b] wraps (bit 0 = x, bit 1 = y) and zeros on the others.  Interior values are rounded as cast_kernel<0> rounds
// them.  Thread = 4 channels of one padded position; c % 4 == 0.
__global__ void pad_cast_kernel(const float* __restrict__ x, int B, int h, int w, int c, const uint8_t* __restrict__ wrap,
                                __half* __restrict__ out) {
    const int nq = c >> 2;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)B * (h + 2) * (w + 2) * nq) return;
    const int q = (int)(i % nq);
    const int64_t pos = i / nq;
    const int pw = w + 2, ph = h + 2;
    const int b = (int)(pos / ((int64_t)ph * pw));
    const int rem = (int)(pos - (int64_t)b * ph * pw);
    int y = rem / pw - 1, xx = rem % pw - 1;
    const int wc = wrap[b];
    bool ok = true;
    if (y < 0 || y >= h) { if (wc & 2) y = wrap_mod(y, h); else ok = false; }
    if (xx < 0 || xx >= w) { if (wc & 1) xx = wrap_mod(xx, w); else ok = false; }
    uint2 pk = make_uint2(0u, 0u);
    if (ok) {
        const float4 v = *(reinterpret_cast<const float4*>(x + (((int64_t)b * h + y) * w + xx) * c) + q);
        pk.x = pack_half2(v.x, v.y);
        pk.y = pack_half2(v.z, v.w);
    }
    *reinterpret_cast<uint2*>(out + pos * c + q * 4) = pk;
}

int launch_pad_cast_f16(const float* x, int B, int h, int w, int c, const uint8_t* wrap, __half* out, cudaStream_t st) {
    ProfScope prof("cast", (double)B * (h + 2) * (w + 2) * c * 6.0, st);
    PB_CHECK(c % 4 == 0 && wrap != nullptr, "pad_cast: c=%d must be a multiple of 4, with a wrap table", c);
    const int64_t n = (int64_t)B * (h + 2) * (w + 2) * (c / 4);
    if (n == 0) return 0;
    pad_cast_kernel<<<ceil_div(n, 256), 256, 0, st>>>(x, B, h, w, c, wrap, out);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_silu_cast_f16(const float* x, int64_t n, __half* out, cudaStream_t st) {
    ProfScope prof("cast", (double)n * 6.0, st);
    if (n == 0) return 0;
    cast_kernel<1><<<ceil_div(ceil_div(n, 4), 256), 256, 0, st>>>(x, nullptr, 1.f, 0.f, n, out);
    PB_LAUNCH_CHECK();
    return 0;
}
int launch_mix_cast_f16(const float* a, const float* b, float wa, float wb, int64_t n, __half* out, cudaStream_t st) {
    ProfScope prof("cast", (double)n * (b ? 10.0 : 6.0), st);
    if (n == 0) return 0;
    cast_kernel<2><<<ceil_div(ceil_div(n, 4), 256), 256, 0, st>>>(a, b, wa, wb, n, out);
    PB_LAUNCH_CHECK();
    return 0;
}
int launch_mix_cast_rows_f16(const float* a, const float* b, const float* w, int64_t per, int64_t n, __half* out, cudaStream_t st) {
    ProfScope prof("cast", (double)n * 10.0, st);
    if (n == 0) return 0;
    PB_CHECK(per >= 4, "mix_cast_rows: %lld elements per weight row (< 4)", (long long)per);
    cast_kernel<3><<<ceil_div(ceil_div(n, 4), 256), 256, 0, st>>>(a, b, 0.f, 0.f, n, out, w, per);
    PB_LAUNCH_CHECK();
    return 0;
}

// Gather + cast of whole samples: packed block j (per elements) is the fp32 block src[j] of `a`, src[j] = samples[j] for
// j < n_list, batch + samples[j - n_list] for the others (a sample's unconditional rows after the batch).  Each element is
// converted as cast_kernel<0> converts it (round to nearest).  per % 4 == 0, so a thread's four elements share one block.
__global__ void gather_cast_kernel(const float* __restrict__ a, const int* __restrict__ samples, int n_list, int batch, int64_t per,
                                   __half* __restrict__ out) {
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= per) return;
    const int j = blockIdx.y;
    const int64_t src = j < n_list ? samples[j] : (int64_t)batch + samples[j - n_list];
    const float4 v = *reinterpret_cast<const float4*>(a + src * per + i);
    uint2 pk;
    pk.x = pack_half2(v.x, v.y);
    pk.y = pack_half2(v.z, v.w);
    *reinterpret_cast<uint2*>(out + (int64_t)j * per + i) = pk;
}

int launch_gather_cast_f16(const float* a, const int* samples, int n_list, int n_blocks, int batch, int64_t per, __half* out,
                           cudaStream_t st) {
    ProfScope prof("cast", (double)n_blocks * per * 6.0, st);
    if (n_blocks == 0 || per == 0) return 0;
    PB_CHECK(per % 4 == 0 && n_blocks <= 65535 && n_blocks <= 2 * n_list, "gather_cast: %d blocks of %lld elements", n_blocks,
             (long long)per);
    dim3 grid((unsigned)ceil_div(ceil_div(per, 4), 256), (unsigned)n_blocks);
    gather_cast_kernel<<<grid, 256, 0, st>>>(a, samples, n_list, batch, per, out);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ tail rows and guidance prompts
// Row gather of a tail: block y copies the `per` bytes of sample src[y] of `base` to sample n_base + y.  V is the widest word
// that divides `per` (the buffers are 256-byte aligned), so each launch moves whole words.
template <typename V>
__global__ void replicate_rows_kernel(uint8_t* __restrict__ base, int64_t words, int n_base, const int* __restrict__ src) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    const int y = blockIdx.y;
    const V* from = reinterpret_cast<const V*>(base) + (int64_t)src[y] * words;
    V* to = reinterpret_cast<V*>(base) + (int64_t)(n_base + y) * words;
    to[i] = from[i];
}

int launch_replicate_rows(void* base, int64_t per, int n_base, const int* src, int n_tail, cudaStream_t st) {
    ProfScope prof("replicate_rows", (double)n_tail * per * 2.0, st);
    if (n_tail == 0 || per == 0) return 0;
    PB_CHECK(src != nullptr && n_tail <= 65535 && ((uintptr_t)base & 15) == 0, "replicate_rows: %d rows", n_tail);
    uint8_t* b = reinterpret_cast<uint8_t*>(base);
    if (per % 16 == 0) {
        replicate_rows_kernel<uint4><<<dim3((unsigned)ceil_div(per / 16, 256), n_tail), 256, 0, st>>>(b, per / 16, n_base, src);
    } else if (per % 4 == 0) {
        replicate_rows_kernel<uint32_t><<<dim3((unsigned)ceil_div(per / 4, 256), n_tail), 256, 0, st>>>(b, per / 4, n_base, src);
    } else {
        replicate_rows_kernel<uint8_t><<<dim3((unsigned)ceil_div(per, 256), n_tail), 256, 0, st>>>(b, per, n_base, src);
    }
    PB_LAUNCH_CHECK();
    return 0;
}

// The K-way guidance mix, in place on fp32 features: composed sample y reads its row of `ld` int32 sample indices [c, u, t_1 ..]
// and `ld` fp32 coefficients, evaluates cast_kernel<3>'s t = fmaf(f_c, a_c, f_u * a_u), then t = fmaf(f_j, a_j, t) in term order
// up to the first index < 0, and writes t over sample c.  per4 = float4 words per sample.
__global__ void __launch_bounds__(256) guidance_mix_kernel(float* __restrict__ f, int64_t per4, const int* __restrict__ rows,
                                                           const float* __restrict__ coef, int ld) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= per4) return;
    const int* idx = rows + (int64_t)blockIdx.y * ld;
    const float* a = coef + (int64_t)blockIdx.y * ld;
    float4* f4 = reinterpret_cast<float4*>(f);
    const float4 c = f4[(int64_t)idx[0] * per4 + i], u = f4[(int64_t)idx[1] * per4 + i];
    const float ac = a[0], au = a[1];
    float4 t = make_float4(fmaf(c.x, ac, u.x * au), fmaf(c.y, ac, u.y * au), fmaf(c.z, ac, u.z * au), fmaf(c.w, ac, u.w * au));
    for (int j = 2; j < ld; ++j) {
        const int s = idx[j];
        if (s < 0) break;
        const float4 v = f4[(int64_t)s * per4 + i];
        const float aj = a[j];
        t = make_float4(fmaf(v.x, aj, t.x), fmaf(v.y, aj, t.y), fmaf(v.z, aj, t.z), fmaf(v.w, aj, t.w));
    }
    f4[(int64_t)idx[0] * per4 + i] = t;
}

int launch_guidance_mix(float* features, int64_t per, const int* rows, const float* coef, int n_composed, int ld, cudaStream_t st) {
    ProfScope prof("guidance_mix", (double)n_composed * per * 4.0 * (ld + 1), st);
    if (n_composed == 0 || per == 0) return 0;
    PB_CHECK(per % 4 == 0 && ld >= 2 && n_composed <= 65535 && ((uintptr_t)features & 15) == 0,
             "guidance_mix: %d samples of %lld elements, %d entries per row", n_composed, (long long)per, ld);
    guidance_mix_kernel<<<dim3((unsigned)ceil_div(per / 4, 256), n_composed), 256, 0, st>>>(features, per / 4, rows, coef, ld);
    PB_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ layout
// [B, R, Cc] -> [B, Cc, R] through a 32x33 shared tile
__global__ void transpose_kernel(const float* __restrict__ in, int R, int Cc, float* __restrict__ out) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const float* src = in + (int64_t)b * R * Cc;
    float* dst = out + (int64_t)b * R * Cc;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        if (r < R && c < Cc) tile[i][threadIdx.x] = src[(int64_t)r * Cc + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (r < R && c < Cc) dst[(int64_t)c * R + r] = tile[threadIdx.x][i];
    }
}

static int transpose(const float* in, int B, int R, int Cc, float* out, cudaStream_t st) {
    if (B == 0 || R == 0 || Cc == 0) return 0;
    dim3 grid(ceil_div(Cc, 32), ceil_div(R, 32), B), block(32, 8);
    PB_CHECK(grid.y <= 65535 && grid.z <= 65535, "transpose: grid too large");
    transpose_kernel<<<grid, block, 0, st>>>(in, R, Cc, out);
    PB_LAUNCH_CHECK();
    return 0;
}

int launch_nchw_to_nhwc(const float* in, int B, int C, int HW, float* out, cudaStream_t st) { return transpose(in, B, C, HW, out, st); }
int launch_nhwc_to_nchw(const float* in, int B, int C, int HW, float* out, cudaStream_t st) { return transpose(in, B, HW, C, out, st); }

// Regional prompts: the mask of every position of every level, the OR of its (patch << level)^2 footprint of token masks.  Output
// level l holds [batch][P_l] at batch * (P_0 + ... + P_{l-1}); sample b reads token-mask row mask_row[b] (NULL: b).
__global__ void __launch_bounds__(256) regional_masks_kernel(const uint8_t* __restrict__ tok, const int* __restrict__ mask_row,
                                                             int batch, int h, int w, int patch, int n_levels, int per_sample,
                                                             uint8_t* __restrict__ out) {
    const int b = blockIdx.y;
    int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= per_sample) return;
    const uint8_t* t = tok + (int64_t)(mask_row ? mask_row[b] : b) * h * w;
    int64_t base = 0;
    for (int l = 0; l < n_levels; ++l) {
        const int s = patch << l, gw = w / s, P = (h / s) * gw;
        if (i < P) {
            const int y = i / gw, x = i - y * gw;
            uint32_t m = 0;
            for (int dy = 0; dy < s; ++dy)
                for (int dx = 0; dx < s; ++dx) m |= t[(y * s + dy) * w + x * s + dx];
            out[base + (int64_t)b * P + i] = (uint8_t)m;
            return;
        }
        i -= P;
        base += (int64_t)batch * P;
    }
}

int launch_regional_masks(const uint8_t* tok_mask, const int* mask_row, int batch, int h, int w, int patch, int n_levels,
                          uint8_t* out, cudaStream_t st) {
    if (batch == 0) return 0;
    int per_sample = 0;
    for (int l = 0; l < n_levels; ++l) per_sample += (h / (patch << l)) * (w / (patch << l));
    ProfScope prof("regional_masks", (double)batch * (n_levels * h * w + per_sample), st);
    PB_CHECK(batch <= 65535, "regional_masks: batch too large");
    regional_masks_kernel<<<dim3(ceil_div(per_sample, 256), batch), 256, 0, st>>>(tok_mask, mask_row, batch, h, w, patch, n_levels,
                                                                                 per_sample, out);
    PB_LAUNCH_CHECK();
    return 0;
}

// Attention maps: one thread per (sample, query position, conditioning key), keys fastest so that the heads' score rows are read
// coalesced.  Every (map row, key, position) has one writer per launch, so the accumulator needs no atomics and a row's sums depend
// on that row alone.
__global__ void __launch_bounds__(256) attention_maps_accumulate_kernel(const AttnParams p, const AttnMapOut mo, float* __restrict__ acc,
                                                                        int acc_ld, int acc_pos, int acc_off) {
    const int b = blockIdx.y;
    const int mr = attn_map_row(mo, b);
    if (mr < 0) return;
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)p.P * p.S_max) return;
    const int pos = (int)(i / p.S_max), s = (int)(i - (int64_t)pos * p.S_max);
    const int slot = p.kv_slot ? p.kv_slot[b] : b;
    const int n_cond = p.kv_len ? p.kv_len[slot] : p.S_max;
    if (s >= n_cond || s >= acc_ld) return;
    const float* sc = mo.scores + ((int64_t)mr * p.nhead * p.P + pos) * p.S_max + s;
    const float* ls = mo.lse2 + (int64_t)mr * p.nhead * p.P + pos;
    float sum = 0.f;
    for (int h = 0; h < p.nhead; ++h) sum += exp2f(sc[(int64_t)h * p.P * p.S_max] - ls[(int64_t)h * p.P]);
    const float* w = nullptr;
    const int n_w = attn_weight_row(p, b, w);
    const int n_self = p.self_attn ? p.P : 0, kj = n_self + s, w_start = n_self + n_cond - n_w;
    if (n_w > 0 && kj >= w_start) sum *= w[kj - w_start];
    acc[((int64_t)mr * acc_ld + s) * acc_pos + acc_off + pos] += sum * (1.0f / (float)p.nhead);
}

int launch_attention_maps_accumulate(const AttnParams& p, const AttnMapOut& mo, float* acc, int acc_ld, int acc_pos, int acc_off,
                                     cudaStream_t st) {
    if (mo.map_batch == 0 || p.P == 0 || p.S_max == 0) return 0;
    ProfScope prof("attention_maps", (double)mo.map_batch * p.P * p.S_max * (p.nhead + 2) * 4.0, st);
    PB_CHECK(mo.map_batch <= 65535, "attention_maps: map batch too large");
    attention_maps_accumulate_kernel<<<dim3((unsigned)ceil_div((int64_t)p.P * p.S_max, 256), mo.map_batch), 256, 0, st>>>(
        p, mo, acc, acc_ld, acc_pos, acc_off);
    PB_LAUNCH_CHECK();
    return 0;
}

// one thread per (row, key, token); the levels are summed in ascending order
__global__ void __launch_bounds__(256) attention_maps_finalize_kernel(const float* __restrict__ acc, int acc_ld, int acc_pos, int S,
                                                                      int h, int w, int patch, int n_levels, float scale,
                                                                      float* __restrict__ maps) {
    const int row = blockIdx.z, s = blockIdx.y;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= h * w) return;
    const int y = i / w, x = i - y * w;
    const float* a = acc + ((int64_t)row * acc_ld + s) * acc_pos;
    float t = 0.f;
    int off = 0;
    for (int l = 0; l < n_levels; ++l) {
        const int st = patch << l, gw = w / st;
        t += a[off + (y / st) * gw + x / st];
        off += (h / st) * gw;
    }
    maps[((int64_t)row * S + s) * h * w + i] = t * scale;
}

int launch_attention_maps_finalize(const float* acc, int rows, int acc_ld, int acc_pos, int S, int h, int w, int patch, int n_levels,
                                   float scale, float* maps, cudaStream_t st) {
    if (rows == 0 || S == 0 || h * w == 0) return 0;
    ProfScope prof("attention_maps", (double)rows * S * h * w * (n_levels + 1) * 4.0, st);
    PB_CHECK(rows <= 65535 && S <= 65535, "attention_maps: %d rows of %d keys", rows, S);
    attention_maps_finalize_kernel<<<dim3(ceil_div(h * w, 256), S, rows), 256, 0, st>>>(acc, acc_ld, acc_pos, S, h, w, patch, n_levels,
                                                                                          scale, maps);
    PB_LAUNCH_CHECK();
    return 0;
}

}  // namespace pb
