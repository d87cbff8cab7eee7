// jsgpu_preview.cu — CimgDecode::CalcChannelPreviewFull beyond its default settings (SURVEY.md §8f N3/N4):
//   * ConvertYCCtoRGB + CapYccRange + CapRgbRange (ImgDecode.cpp:4229-4601), the clipping/histogram colour conversion the
//     reference takes when CSnoopConfig::bHistoEn or bStatClipEn is set (:4745), with its statistics: m_sHisto (min/max/sum of
//     the twelve channels), m_sStatClip, m_anCcHisto_r/g/b, m_anHistoYFull and the capped "YCC Clipped" notes;
//   * ChannelExtract (:4832-4876), the eight preview modes;
//   * the YCC level shift from a given MCU on (:4735-4739).
// The default settings never come here: the fused IDCT kernel has written exactly that DIB already.
//
// One pass over the pixel maps (6 B/px read, 4 B/px written): a CTA takes whole pixel rows of one image, keeps the histograms
// in shared memory and the ranges in registers, and leaves per-row counts of YCC clip events behind; k_preview_warn then
// reproduces the reference's "first YCC_CLIP_REPORT_MAX notes, and only those are counted" rule (:4372-4378) by walking, in
// raster order, just the rows that have events.
#include "jsgpu_internal.h"
#include "jsgpu_ycc.cuh"

#define FULL 0xffffffffu
#define PV_THREADS 256

struct PvPix {                       // PixelCc (ImgDecode.h:186-216), the fields that are used
    int pre_y, pre_cb, pre_cr;       // nPrerangeY/Cb/Cr
    int rng_y, rng_cb, rng_cr;       // nPreclipY/Cb/Cr (after ranging, before the clip)
    uint32_t fy, fcb, fcr;           // nFinalY/Cb/Cr
    int pr, pg, pb;                  // (int)nPreclipR/G/B
    uint32_t fr, fg, fb;             // nFinalR/G/B
};

// ConvertYCCtoRGBFastFloat (ImgDecode.cpp:4086-4139)
__device__ __forceinline__ void pv_fast(PvPix& p)
{
    const YccFast o = ycc_fast(p.pre_y, p.pre_cb, p.pre_cr);
    p.fy = (uint32_t)(o.y + 128); p.fcb = (uint32_t)(o.cb + 128); p.fcr = (uint32_t)(o.cr + 128);
    p.fr = o.r; p.fg = o.g; p.fb = o.b;
}

// ConvertYCCtoRGB without its bookkeeping (:4229-4325): ranging (C division, truncating), YCC clip, conversion, RGB clip
__device__ __forceinline__ void pv_full(PvPix& p)
{
    p.rng_y = (p.pre_y + 1024) / 8; p.rng_cb = (p.pre_cb + 1024) / 8; p.rng_cr = (p.pre_cr + 1024) / 8;
    const int y = max(0, min(255, p.rng_y)), cb = max(0, min(255, p.rng_cb)), cr = max(0, min(255, p.rng_cr));
    p.fy = (uint32_t)y; p.fcb = (uint32_t)cb; p.fcr = (uint32_t)cr;
    float vr, vg, vb; ycc_float_core((float)(y - 128), (float)(cb - 128), (float)(cr - 128), vr, vg, vb);
    p.pr = __float2int_rz(vr); p.pg = __float2int_rz(vg); p.pb = __float2int_rz(vb);
    p.fr = (uint32_t)max(0, min(255, p.pr)); p.fg = (uint32_t)max(0, min(255, p.pg)); p.fb = (uint32_t)max(0, min(255, p.pb));
}

// ChannelExtract (:4832-4876): the DIB word [B,G,R,0]
__device__ __forceinline__ uint32_t pv_extract(int mode, const PvPix& p)
{
    uint32_t r = p.fr, g = p.fg, b = p.fb;
    switch (mode) {
    case 2: r = p.fcr; g = p.fy; b = p.fcb; break;          // PREVIEW_YCC
    case 3: g = b = p.fr; break;                            // PREVIEW_R
    case 4: r = b = p.fg; break;
    case 5: r = g = p.fb; break;
    case 6: r = g = b = p.fy; break;                        // PREVIEW_Y
    case 7: r = g = b = p.fcb; break;
    case 8: r = g = b = p.fcr; break;
    default: break;                                         // PREVIEW_RGB and anything else
    }
    return b | (g << 8) | (r << 16);
}

__device__ __forceinline__ bool pv_shifted(const DevImage& im, const jsgpu_preview& pv, uint32_t px, uint32_t py)
{
    // nMcuInd >= nMcuShiftInd (:4733-4739); both use m_nImgSizeX / m_nMcuWidth MCUs per row
    return (py / im.mcu_h) * im.mcu_xmax + px / im.mcu_w >= pv.shift_mcu_y * im.mcu_xmax + pv.shift_mcu_x;
}
__device__ __forceinline__ void pv_load(const DevBatch& b, const DevImage& im, const jsgpu_preview& pv, uint32_t px, uint32_t py, PvPix& p)
{
    const size_t i = im.pix_off + (size_t)py * im.wp + px;
    p.pre_y = b.pix_y[i]; p.pre_cb = 0; p.pre_cr = 0;
    if (im.ns == 3) { p.pre_cb = b.pix_cb[i]; p.pre_cr = b.pix_cr[i]; }
    if (pv_shifted(im, pv, px, py)) { p.pre_y += pv.shift_y; p.pre_cb += pv.shift_cb; p.pre_cr += pv.shift_cr; }
}

#define PV_CC_COPIES 8               // copies of the 3 x 128-bin colour histograms: neighbouring pixels mostly fall into the same bin,
struct PvShared {                    // so the lanes of a warp are spread over copies to keep their shared-memory atomics apart
    uint32_t cc[PV_CC_COPIES][3][JSGPU_CC_HISTO_BINS];
    uint32_t yh[JSGPU_Y_HISTO_BINS];
};

// Four pixels per thread (the map width is a multiple of 8 and an MCU at least 8 wide, so a group of four never straddles a row or an
// MCU): 8-byte loads from the three maps, one 16-byte store into the DIB.
template <bool FULLCONV, bool HIST>
__global__ void __launch_bounds__(PV_THREADS) k_preview(DevBatch b, jsgpu_preview pv, jsgpu_colour_stats* st, uint32_t* rowclip)
{
    __shared__ PvShared sh;
    // one image per blockIdx.y, strided beyond 65535 images: a CTA that moves on flushes its histograms and ranges first and
    // starts the next image from zero
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
    const DevImage& im = b.img[ii];
    if (!im.valid) continue;
    if (HIST) { __syncthreads(); for (uint32_t i = threadIdx.x; i < sizeof(PvShared) / 4; i += PV_THREADS) reinterpret_cast<uint32_t*>(&sh)[i] = 0; __syncthreads(); }
    int vmin[12], vmax[12]; long long vsum[12]; uint32_t rgbclip[6];
    #pragma unroll
    for (int k = 0; k < 12; k++) { vmin[k] = 0; vmax[k] = 0; vsum[k] = 0; }     // memset(&m_sHisto, 0) (:3147): the ranges START at 0
    #pragma unroll
    for (int k = 0; k < 6; k++) rgbclip[k] = 0;
    unsigned long long sum_fy = 0, npx = 0;
    uint32_t (*const mycc)[JSGPU_CC_HISTO_BINS] = sh.cc[threadIdx.x & (PV_CC_COPIES - 1)];
    for (uint32_t py = blockIdx.x; py < im.hp; py += gridDim.x) {
        uint32_t row_events = 0;
        const size_t row = im.pix_off + (size_t)py * im.wp;
        uint4* const drow = reinterpret_cast<uint4*>(b.dib + im.dib_off + (size_t)(im.hp - 1 - py) * im.wp * 4);     // bottom-up (:4786-4789)
        for (uint32_t px = threadIdx.x * 4; px < im.wp; px += PV_THREADS * 4) {
            const short4 vy = *reinterpret_cast<const short4*>(b.pix_y + row + px);
            short4 vb = make_short4(0, 0, 0, 0), vr = vb;
            if (im.ns == 3) { vb = *reinterpret_cast<const short4*>(b.pix_cb + row + px); vr = *reinterpret_cast<const short4*>(b.pix_cr + row + px); }
            const bool sh_on = pv_shifted(im, pv, px, py);
            const bool det = pv.detail_en && px / im.mcu_w == pv.detail_mcu_x && py / im.mcu_h == pv.detail_mcu_y;
            const int sy = sh_on ? pv.shift_y : 0, sb = sh_on ? pv.shift_cb : 0, sr = sh_on ? pv.shift_cr : 0;
            const int y4[4] = { vy.x, vy.y, vy.z, vy.w }, b4[4] = { vb.x, vb.y, vb.z, vb.w }, r4[4] = { vr.x, vr.y, vr.z, vr.w };
            uint32_t o[4];
            #pragma unroll
            for (int q = 0; q < 4; q++) {
                PvPix p; p.pre_y = y4[q] + sy; p.pre_cb = b4[q] + sb; p.pre_cr = r4[q] + sr;
                if (FULLCONV) {
                    pv_full(p);
                    row_events += (p.rng_y > 255) + (p.rng_y < 0) + (p.rng_cb > 255) + (p.rng_cb < 0) + (p.rng_cr > 255) + (p.rng_cr < 0);
                    rgbclip[0] += p.pr < 0; rgbclip[1] += p.pr > 255; rgbclip[2] += p.pg < 0; rgbclip[3] += p.pg > 255; rgbclip[4] += p.pb < 0; rgbclip[5] += p.pb > 255;
                    if (HIST) {
                        const int v[12] = { p.pre_y, p.pre_cb, p.pre_cr, p.rng_y, p.rng_cb, p.rng_cr, p.pr, p.pg, p.pb, (int)p.fr, (int)p.fg, (int)p.fb };
                        #pragma unroll
                        for (int k = 0; k < 12; k++) { vmin[k] = min(vmin[k], v[k]); vmax[k] = max(vmax[k], v[k]); vsum[k] += v[k]; }
                        npx++;
                        atomicAdd(&sh.yh[max(-1024, min(1023, p.pre_y)) + 1024], 1u);              // m_anHistoYFull (:4251-4260)
                        atomicAdd(&mycc[0][p.fr >> 1], 1u); atomicAdd(&mycc[1][p.fg >> 1], 1u); atomicAdd(&mycc[2][p.fb >> 1], 1u);   // 256 / HISTO_BINS = 2 (:4313-4321)
                    }
                } else pv_fast(p);
                sum_fy += p.fy;
                o[q] = pv_extract(pv.mode, p);
                if (det) st[ii].detail_rgb[py - pv.detail_mcu_y * im.mcu_h][px + q - pv.detail_mcu_x * im.mcu_w] = (p.fr << 16) | (p.fg << 8) | p.fb;   // sPixSrc.nFinalR/G/B (:4763)
            }
            drow[px >> 2] = make_uint4(o[0], o[1], o[2], o[3]);
        }
        if (FULLCONV) {
            row_events = __reduce_add_sync(FULL, row_events);
            if ((threadIdx.x & 31) == 0 && row_events) atomicAdd(&rowclip[im.row_off + py], row_events);
        }
    }
    jsgpu_colour_stats* const o = st + ii;
    for (int d = 16; d; d >>= 1) sum_fy += __shfl_xor_sync(FULL, sum_fy, d);
    if ((threadIdx.x & 31) == 0 && sum_fy) atomicAdd(&b.sum_y[ii], sum_fy);
    if (FULLCONV) {
        #pragma unroll
        for (int k = 0; k < 6; k++) {
            const uint32_t t = __reduce_add_sync(FULL, rgbclip[k]);
            if ((threadIdx.x & 31) == 0 && t) atomicAdd(&o->clip[6 + k], t);
        }
    }
    if (HIST) {
        #pragma unroll
        for (int k = 0; k < 12; k++) {
            const int mn = __reduce_min_sync(FULL, vmin[k]), mx = __reduce_max_sync(FULL, vmax[k]);
            long long s = vsum[k];
            for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(FULL, s, d);
            if ((threadIdx.x & 31) == 0) {
                if (mn < 0) atomicMin(&o->vmin[k], mn);
                if (mx > 0) atomicMax(&o->vmax[k], mx);
                if (s) atomicAdd(reinterpret_cast<unsigned long long*>(&o->vsum[k]), (unsigned long long)s);
            }
        }
        for (int d = 16; d; d >>= 1) npx += __shfl_xor_sync(FULL, npx, d);
        if ((threadIdx.x & 31) == 0 && npx) atomicAdd(reinterpret_cast<unsigned long long*>(&o->count), npx);
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < 3 * JSGPU_CC_HISTO_BINS; i += PV_THREADS) {
            uint32_t v = 0;
            #pragma unroll
            for (int c = 0; c < PV_CC_COPIES; c++) v += (&sh.cc[c][0][0])[i];
            if (v) atomicAdd(&o->cc_histo[0][0] + i, v);
        }
        for (uint32_t i = threadIdx.x; i < JSGPU_Y_HISTO_BINS; i += PV_THREADS) { const uint32_t v = sh.yh[i]; if (v) atomicAdd(&o->y_histo[i], v); }
    }
    }
}

// CapYccRange's notes (:4366-4466): the first `ycc_warn_budget` clip events in raster order, each counted in m_sStatClip only
// while notes are still being issued.  One warp per image: the lanes look for rows with events, lane 0 walks them.
__global__ void __launch_bounds__(32) k_preview_warn(DevBatch b, jsgpu_preview pv, jsgpu_colour_stats* st, const uint32_t* rowclip)
{
    const DevImage& im = b.img[blockIdx.x];
    if (!im.valid) return;
    jsgpu_colour_stats* const o = st + blockIdx.x;
    const uint32_t lane = threadIdx.x, budget = min(pv.ycc_warn_budget, (uint32_t)JSGPU_MAX_YCC_WARN);
    uint32_t nwarn = 0;
    for (uint32_t r0 = 0; r0 < im.hp && nwarn < budget; r0 += 32) {
        const uint32_t r = r0 + lane;
        uint32_t rows = __ballot_sync(FULL, r < im.hp && rowclip[im.row_off + r] != 0);
        while (rows && nwarn < budget) {
            const uint32_t py = r0 + (uint32_t)__ffs(rows) - 1; rows &= rows - 1;
            if (lane == 0) {
                for (uint32_t px = 0; px < im.wp && nwarn < budget; px++) {
                    PvPix p; pv_load(b, im, pv, px, py, p);
                    int cy = (p.pre_y + 1024) / 8, ccb = (p.pre_cb + 1024) / 8, ccr = (p.pre_cr + 1024) / 8;
                    // the order of the checks and the running values the notes print: Y over, Y under, Cb over, Cb under, Cr over, Cr under
                    #pragma unroll
                    for (int k = 0; k < 6; k++) {
                        int& cur = (k < 2) ? cy : (k < 4) ? ccb : ccr;
                        const bool over = !(k & 1);
                        if (over ? (cur > 255) : (cur < 0)) {
                            if (nwarn < budget) {
                                jsgpu_ycc_warn& w = o->warn[nwarn++];
                                w.mcu_x = px / im.mcu_w; w.mcu_y = py / im.mcu_h; w.y = cy; w.cb = ccb; w.cr = ccr; w.px = px; w.py = py;
                                w.kind = (uint32_t)((k & ~1) + (over ? 1 : 0));                // clip[]: under, over per channel
                                o->clip[w.kind]++;
                            }
                            cur = over ? 255 : 0;
                        }
                    }
                }
            }
            nwarn = __shfl_sync(FULL, nwarn, 0);
        }
    }
    if (lane == 0) o->nwarn = nwarn;
}

// stats[] after a preview pass: m_nAvgY = nSumY / nNumPixels with nSumY an `unsigned` (wraps) and
// nNumPixels = (Y+1)*(X+1) (ImgDecode.cpp:4633,4689,4813-4818)
__global__ void k_preview_stats(DevBatch b)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.nimg) return;
    const DevImage& im = b.img[i];
    if (!im.valid) return;
    const unsigned long long s = b.sum_y[i];
    int32_t* st = b.stats + (size_t)i * JSGPU_STAT_WORDS;
    st[JSGPU_STAT_SUMY_LO] = (int32_t)(uint32_t)s; st[JSGPU_STAT_SUMY_HI] = (int32_t)(uint32_t)(s >> 32);
    const unsigned long npix = (unsigned long)(im.hp + 1) * (unsigned long)(im.wp + 1);
    st[JSGPU_STAT_AVGY] = (int32_t)((unsigned long)(uint32_t)s / (npix ? npix : 1ul));
}

int js_launch_preview(const DevBatch& b, const jsgpu_preview& pv, jsgpu_colour_stats* st, uint32_t* rowclip, uint64_t rows_total,
                      uint32_t max_hp, int sm_count, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    const bool full = pv.hist_en || pv.statclip_en, hist = pv.hist_en != 0;
    cudaMemsetAsync(st, 0, sizeof(jsgpu_colour_stats) * (size_t)b.nimg, s);
    cudaMemsetAsync(b.sum_y, 0, sizeof(unsigned long long) * (size_t)b.nimg, s);
    if (full) cudaMemsetAsync(rowclip, 0, sizeof(uint32_t) * (size_t)rows_total, s);
    // enough CTAs per image to fill the device whatever the batch size, never more than its rows
    uint32_t per_img = (uint32_t)((sm_count * 8 + b.nimg - 1) / b.nimg);
    if (per_img > max_hp) per_img = max_hp;
    if (per_img < 1) per_img = 1;
    const dim3 grid(per_img, b.nimg < 65535u ? b.nimg : 65535u);
    int n = 0;
    if (full && hist) k_preview<true, true><<<grid, PV_THREADS, 0, s>>>(b, pv, st, rowclip);
    else if (full)    k_preview<true, false><<<grid, PV_THREADS, 0, s>>>(b, pv, st, rowclip);
    else              k_preview<false, false><<<grid, PV_THREADS, 0, s>>>(b, pv, st, rowclip);
    n++;
    if (full && pv.ycc_warn_budget) { k_preview_warn<<<b.nimg, 32, 0, s>>>(b, pv, st, rowclip); n++; }
    k_preview_stats<<<(b.nimg + 127) / 128, 128, 0, s>>>(b);
    return n + 1;
}

// ---- Export-to-TIFF consumer (SURVEY.md §8f N4) ---------------------------------------------------------------------------
// The three-samples-per-pixel, top-down array CJPEGsnoopDoc::OnToolsExporttiff builds before FileTiff::WriteFile
// (JPEGsnoopDoc.cpp:2108-2170), packed on the device so that 3 (or 6) bytes per pixel cross the bus instead of the DIB's 4 or
// the pixel maps' 6.  Four pixels per thread: the image width is a multiple of 8, so a group never straddles a row.
template <int MODE>
__global__ void __launch_bounds__(256) k_export_pack(DevBatch b, uint32_t image, uint8_t* out)
{
    const DevImage& im = b.img[image];
    const uint32_t groups_per_row = im.wp >> 2;
    const uint64_t ngroups = (uint64_t)groups_per_row * im.hp;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t py = (uint32_t)(g / groups_per_row), px = (uint32_t)(g % groups_per_row) * 4;
        uint32_t s[12];                                              // R,G,B (or Y,Cb,Cr) of the four pixels, 0..255
        if (MODE == JSGPU_EXPORT_YCC8) {
            // clip to -1024..1023, then (0x400 + v) >> 3 (:2150-2166)
            const size_t i = im.pix_off + (size_t)py * im.wp + px;
            const short4 vy = *reinterpret_cast<const short4*>(b.pix_y + i), vb = *reinterpret_cast<const short4*>(b.pix_cb + i),
                         vr = *reinterpret_cast<const short4*>(b.pix_cr + i);
            const short y4[4] = { vy.x, vy.y, vy.z, vy.w }, b4[4] = { vb.x, vb.y, vb.z, vb.w }, r4[4] = { vr.x, vr.y, vr.z, vr.w };
            #pragma unroll
            for (int k = 0; k < 4; k++) {
                s[k * 3 + 0] = (uint32_t)(0x400 + max(-1024, min(1023, (int)y4[k]))) >> 3;
                s[k * 3 + 1] = (uint32_t)(0x400 + max(-1024, min(1023, (int)b4[k]))) >> 3;
                s[k * 3 + 2] = (uint32_t)(0x400 + max(-1024, min(1023, (int)r4[k]))) >> 3;
            }
        } else {
            // the DIB is bottom-up, [B,G,R,0] (:2112-2116)
            const uint4 d = *reinterpret_cast<const uint4*>(b.dib + im.dib_off + ((size_t)(im.hp - 1 - py) * im.wp + px) * 4);
            const uint32_t w[4] = { d.x, d.y, d.z, d.w };
            #pragma unroll
            for (int k = 0; k < 4; k++) { s[k * 3 + 0] = (w[k] >> 16) & 0xFF; s[k * 3 + 1] = (w[k] >> 8) & 0xFF; s[k * 3 + 2] = w[k] & 0xFF; }
        }
        if (MODE == JSGPU_EXPORT_RGB16) {
            // Swap16(v << 8) stored as an unsigned short (:2125-2129): bytes v, 0 — the big-endian sample v * 256
            uint32_t* o = reinterpret_cast<uint32_t*>(out + g * 24);
            #pragma unroll
            for (int k = 0; k < 6; k++) o[k] = s[2 * k] | (s[2 * k + 1] << 16);
        } else {
            uint32_t* o = reinterpret_cast<uint32_t*>(out + g * 12);
            #pragma unroll
            for (int k = 0; k < 3; k++) o[k] = s[4 * k] | (s[4 * k + 1] << 8) | (s[4 * k + 2] << 16) | (s[4 * k + 3] << 24);
        }
    }
}

int js_launch_export(const DevBatch& b, uint32_t image, int mode, uint8_t* out, uint64_t npx, int sm_count, cudaStream_t s)
{
    uint64_t want = (npx / 4 + 255) / 256;
    const uint32_t grid = (uint32_t)(want < (uint64_t)sm_count * 8 ? (want ? want : 1) : (uint64_t)sm_count * 8);
    if (mode == JSGPU_EXPORT_RGB16)     k_export_pack<JSGPU_EXPORT_RGB16><<<grid, 256, 0, s>>>(b, image, out);
    else if (mode == JSGPU_EXPORT_YCC8) k_export_pack<JSGPU_EXPORT_YCC8><<<grid, 256, 0, s>>>(b, image, out);
    else                                k_export_pack<JSGPU_EXPORT_RGB8><<<grid, 256, 0, s>>>(b, image, out);
    return 1;
}
