// jsgpu_api.cu — the C-ABI of include/jsgpu.h: context, table upload, batch planning
// (geometry / validation / allocation of ImgDecode.cpp:2755-3123 for n images), and the
// enqueue of the kernels in jsgpu_kernels.cu.  No CPU decode path exists here: every
// decode goes to the device or fails.
#include "../../include/jsgpu.h"
#include "jsgpu_internal.h"
#include "jsgpu_tables_host.h"
#include "jsgpu_phuff_core.cuh"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdarg>
#include <string>
#include <vector>
#include <memory>
#include <array>
#include <algorithm>
#include <dlfcn.h>

#define JSGPU_VERSION 100

// Lays out consecutive arrays in one pool.  Run once with base == nullptr to measure the bytes to reserve, then on the
// reserved block to bind the pointers; align(a) counts a whole `a` bytes while measuring (the most it can skip).
struct Carve {
    uint8_t* base; size_t off = 0;
    template <class T> void take(T*& p, uint64_t n) { p = base ? (T*)(base + off) : nullptr; off += n * sizeof(T); }
    void align(size_t a) { off = base ? (off + a - 1) / a * a : off + a; }
    void skip(size_t bytes) { off += bytes; }
};
template <class Layout> static cudaError_t carve(DevBuf& pool, Layout lay)
{
    Carve m{nullptr}; lay(m);
    const cudaError_t e = pool.reserve(m.off);
    if (e == cudaSuccess) { Carve c{(uint8_t*)pool.p}; lay(c); }
    return e;
}

// Everything jsgpu_batch_begin derives from the image descriptors, on the host (plan_batch).
struct BatchPlan {
    std::vector<DevImage> img;
    std::vector<jsgpu_image_layout> layout;
    std::vector<uint2> items;                // Huffman warp kernel: [all | without self-synchronised images]
    std::vector<uint2> litems;               // lane kernel: [all | without ... | slots of the self-synchronised images]
    uint32_t n_items = 0, n_items_np = 0, n_litems = 0, n_litems_np = 0, n_vitems = 0;
    std::vector<uint4> tiles;                // fused IDCT tiles grouped by chroma replication class
    uint32_t tcls_first[3] = {}, tcls_count[3] = {}, plane_bytes = 0;
    std::vector<uint32_t> mc_img;            // image of every 4096-byte chunk (marker scan)
    // pool totals in elements (pix, blk: int16; dib: bytes; mcu, histo, stats: words), and the other sizes of the batch
    uint64_t bits_len = 0, pix = 0, dib = 0, blk = 0, mcu = 0, histo = 0, stats = 0;
    uint64_t coef_rows = 0, max_scan_len = 0, ubits = 0, ph = 0, rt = 0, cs = 0, rows = 0;
    uint32_t nseg = 0, nseg_np = 0, n_psync = 0, max_cs = 0, max_hp = 0, n_std = 0, n_nonstd = 0;
};

// What the context holds of its batch.  The order matters: from JS_PLANNED on the device pools are bound.
enum BatchState {
    JS_NO_BATCH,
    JS_LAYOUT_ONLY,     // the chunked jsgpu_decode_batch_host: layout and statuses here, the device pools are the chunk contexts'
    JS_PLANNED,         // jsgpu_batch_begin: pools reserved and bound
    JS_DECODED,         // jsgpu_batch_decode: the outputs are resident on the device
};

struct jsgpu_ctx {
    int device = 0, sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t stream2 = nullptr;          // MCU-file-map kernels run here, next to the IDCT kernel
    cudaEvent_t evx[2] = {};
    cudaEvent_t ev[6] = {};
    cudaEvent_t tev[2] = {};
    std::string err;
    jsgpu_options opt;
    bool have_idct = false;
    // device state
    DevBuf d_ctab; bool have_ctab = false;
    DevBuf d_li, d_lf, d_sym, d_tables, d_img, d_items, d_litems, d_tiles, d_ubits, d_seg64, d_ph, d_rowtab, d_ex;
    bool sym_ok = false, baked_ok = false, bakedf_ok = false, tab_baked = false;
    DevBuf d_bits, d_seg, d_coef, d_mcubits, d_pix, d_dib, d_blk, d_mcumap, d_histo, d_stats, d_misc;
    uint32_t nsets = 0;
    std::vector<std::array<uint32_t, JS_NSLOT>> set_l2;   // per table set and slot: second-level entries used (0xffffffff = overflowed)
    // batch state
    BatchState state = JS_NO_BATCH;
    BatchPlan plan;
    DevBatch batch;
    int launches = 0;
    // host copies of the configuration, replayed into the chunk contexts of jsgpu_decode_batch_host
    std::vector<jsgpu_tables> h_sets; std::vector<int32_t> h_li; std::vector<float> h_lf;
    std::vector<jsgpu_ctx*> kids;            // chunk contexts (own stream and pools), created on first use
    // CalcChannelPreviewFull settings (jsgpu_set_preview) and the statistics of the last preview pass
    jsgpu_preview pv = {0, 0, 1, 0, 0, 0, 0, 0, JSGPU_MAX_YCC_WARN, 0, 0, 0, 0};
    DevBuf d_mc;                             // marker-scan chunk arrays
    DevBuf d_cstats, d_rowclip; bool pv_done = false;
    // "Detailed Decode" request (jsgpu_set_detail) and the dump of the last decode
    jsgpu_detail dtl = {0, 0, 0, 0, 0}; bool dt_done = false;
    DevBuf d_dt_ev, d_dt_mat;                // events and matrices, sized at each decode
    DevBuf d_dt_scratch;                     // [16] counters (JsDetailOut::hdr), [JSGPU_HISTO_WORDS] the walk's code-length histogram, then the
                                             // parallel path's per-MCU event counts / offsets and last top-up points
    bool dt_parallel = false; JsDetailRange dt_range = {0, 0, 0, 0, 0}; JsDetailOut dt_out = {};
    uint32_t scan_warn_start = 0; bool scan_errors_disable = false;      // jsgpu_set_scan_error_state
    JsErrCfg ex_cfg = {20, 0, 0};            // the error report's settings of the last decode (an events-only walk repeats them)
    DevBuf d_ex_all;                         // jsgpu_batch_error_events: the walk's result and histogram scratch, then every event
    JsSearch* search = nullptr;              // jsgpu_search_bytes: own streams, staging and device buffers (not the batch pools)
};

static int vfail(std::string& err, int code, const char* fmt, va_list ap)
{
    char buf[512];
    vsnprintf(buf, sizeof buf, fmt, ap);
    err = buf;
    return code;
}
static int fail(std::string& err, int code, const char* fmt, ...) { va_list ap; va_start(ap, fmt); vfail(err, code, fmt, ap); va_end(ap); return code; }
static int fail(jsgpu_ctx* c, int code, const char* fmt, ...) { va_list ap; va_start(ap, fmt); vfail(c->err, code, fmt, ap); va_end(ap); return code; }
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(ctx, (e_ == cudaErrorMemoryAllocation) ? JSGPU_ENOMEM : JSGPU_ECUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); } while (0)
static const char* const HOST_DELIVERED = "the last batch was delivered to host buffers by jsgpu_decode_batch_host";

// The ten per-image outputs, indexed by JSGPU_OUT_*.  A pool holds the images back to back in batch order: image i's
// elements start at its DevImage offset `off`, or at i * count for the fixed-size outputs (off == nullptr).
struct JsOutput {
    size_t dev, host;                            // offsetof its pool pointer in DevBatch and in jsgpu_host_outputs (= jsgpu_pools)
    uint32_t elem;                               // bytes per element
    bool chroma;                                 // absent from a one-component scan
    uint64_t DevImage::* off;
    uint64_t (*count)(const DevImage& im);       // elements of one image
    uint64_t BatchPlan::* total;                 // elements of the pool
};
static uint64_t js_npx(const DevImage& im) { return (uint64_t)im.wp * im.hp; }
static uint64_t js_nblk(const DevImage& im) { return (uint64_t)im.blk_xmax * im.blk_ymax; }
#define JS_OUT(f, hf, elem, chroma, off, count, total) { offsetof(DevBatch, f), offsetof(jsgpu_host_outputs, hf), elem, chroma, off, count, &BatchPlan::total }
static const JsOutput js_outputs[] = {
    JS_OUT(pix_y,   pix_y,     2, false, &DevImage::pix_off, js_npx, pix),
    JS_OUT(pix_cb,  pix_cb,    2, true,  &DevImage::pix_off, js_npx, pix),
    JS_OUT(pix_cr,  pix_cr,    2, true,  &DevImage::pix_off, js_npx, pix),
    JS_OUT(dib,     dib,       1, false, &DevImage::dib_off, [](const DevImage& im) { return js_npx(im) * 4; }, dib),
    JS_OUT(blk_y,   blk_y,     2, false, &DevImage::blk_off, js_nblk, blk),
    JS_OUT(blk_cb,  blk_cb,    2, true,  &DevImage::blk_off, js_nblk, blk),
    JS_OUT(blk_cr,  blk_cr,    2, true,  &DevImage::blk_off, js_nblk, blk),
    JS_OUT(mcu_map, mcu_map,   4, false, &DevImage::mcu_off, [](const DevImage& im) -> uint64_t { return im.nmcu; }, mcu),
    JS_OUT(histo,   dht_histo, 4, false, nullptr, [](const DevImage&) -> uint64_t { return JSGPU_HISTO_WORDS; }, histo),
    JS_OUT(stats,   stats,     4, false, nullptr, [](const DevImage&) -> uint64_t { return JSGPU_STAT_WORDS; }, stats),
};
#undef JS_OUT
static_assert(sizeof js_outputs / sizeof js_outputs[0] == JSGPU_OUT_STATS + 1, "one entry per JSGPU_OUT_* selector");
static_assert(offsetof(jsgpu_pools, stats) == offsetof(jsgpu_host_outputs, stats), "the ten outputs lead both structs");
static uint64_t out_off(const JsOutput& o, const DevImage& im, uint32_t i) { return o.off ? im.*o.off : i * o.count(im); }
static void* get_ptr(const void* s, size_t off) { void* p; memcpy(&p, (const uint8_t*)s + off, sizeof p); return p; }
static void set_ptr(void* s, size_t off, void* p) { memcpy((uint8_t*)s + off, &p, sizeof p); }

static bool preview_is_default(const jsgpu_preview& p)
{
    return !p.hist_en && !p.statclip_en && (p.mode == 0 || p.mode == 1) && !p.shift_y && !p.shift_cb && !p.shift_cr;
}
static int run_preview(jsgpu_ctx* ctx, const jsgpu_preview& pv, int* launches)
{
    const size_t n = ctx->plan.img.size();
    CK(ctx->d_cstats.reserve(n * sizeof(jsgpu_colour_stats)));
    CK(ctx->d_rowclip.reserve((size_t)ctx->plan.rows * 4 + 16));
    *launches += js_launch_preview(ctx->batch, pv, (jsgpu_colour_stats*)ctx->d_cstats.p, (uint32_t*)ctx->d_rowclip.p, ctx->plan.rows,
                                   ctx->plan.max_hp, ctx->sm_count, ctx->stream);
    ctx->pv_done = true;
    return JSGPU_OK;
}

extern "C" {

int jsgpu_version(void) { return JSGPU_VERSION; }

const char* jsgpu_strerror(int code)
{
    switch (code) {
    case JSGPU_OK: return "ok";
    case JSGPU_ENODEV: return "no usable CUDA device";
    case JSGPU_EINVAL: return "invalid argument";
    case JSGPU_ENOMEM: return "out of memory";
    case JSGPU_ECUDA: return "CUDA error";
    case JSGPU_ESTATE: return "call out of order";
    case JSGPU_EUNSUP: return "image not supported by the scan decoder";
    default: return "unknown error";
    }
}
const char* jsgpu_last_error(const jsgpu_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int jsgpu_init(int device, jsgpu_ctx** out)
{
    if (!out) return JSGPU_EINVAL;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return JSGPU_ENODEV;       // no CPU fallback by design
    if (device < 0 || device >= ndev) return JSGPU_EINVAL;
    if (cudaSetDevice(device) != cudaSuccess) return JSGPU_ENODEV;
    jsgpu_ctx* ctx = new jsgpu_ctx();
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return JSGPU_ENODEV; }
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return JSGPU_ECUDA; }
    if (cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking) != cudaSuccess) { cudaStreamDestroy(ctx->stream); delete ctx; return JSGPU_ECUDA; }
    for (auto& ev : ctx->evx) cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    for (auto& ev : ctx->ev) cudaEventCreate(&ev);
    for (auto& ev : ctx->tev) cudaEventCreate(&ev);
    memset(&ctx->opt, 0, sizeof ctx->opt);
    ctx->opt.decode_ac = 1; ctx->opt.want_histo = 1; ctx->opt.want_mcu_map = 1; ctx->opt.device_markers = 1;
    ctx->opt.scan_err_max = 20;                          // CSnoopConfig::nErrMaxDecodeScan's default (SnoopConfig.cpp:89)
    memset(&ctx->batch, 0, sizeof ctx->batch);
    *out = ctx;
    return JSGPU_OK;
}

void jsgpu_free(jsgpu_ctx* ctx)
{
    if (!ctx) return;
    for (jsgpu_ctx* k : ctx->kids) jsgpu_free(k);
    ctx->kids.clear();
    js_search_free(ctx->search);
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto& ev : ctx->ev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->tev) if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->evx) if (ev) cudaEventDestroy(ev);
    if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

void* jsgpu_stream(jsgpu_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int jsgpu_sync(jsgpu_ctx* ctx)
{
    if (!ctx) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

// Split the integer IDCT table into its mirror-symmetric part (quadrant y,x < 4) and a sparse
// correction: Li[y][x][vu] = sy*sx*S[min(y,7-y)][min(x,7-x)][vu] + D[yx][vu], sx = (x>=4 && u odd) ? -1 : 1,
// sy = (y>=4 && v odd) ? -1 : 1.  Usable by the fused kernel when D is non-zero for <= 4 values of vu.
static bool build_idct_sym(const int32_t* li, IdctSym& sym)
{
    memset(&sym, 0, sizeof sym);
    std::vector<int> pos;
    for (int vu = 0; vu < 64; vu++) {
        const int u = vu & 7, v = vu >> 3;
        bool any = false;
        for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) {
            const int yy = y < 4 ? y : 7 - y, xx = x < 4 ? x : 7 - x;
            int sg = 1; if (x >= 4 && (u & 1)) sg = -sg; if (y >= 4 && (v & 1)) sg = -sg;
            const int d = li[(y * 8 + x) * 64 + vu] - sg * li[(yy * 8 + xx) * 64 + vu];
            if (d != 0 && vu >= 1) any = true;
        }
        for (int q = 0; q < 16; q++) sym.s4[vu][q >> 2][q & 3] = li[((q >> 2) * 8 + (q & 3)) * 64 + vu];
        if (any) pos.push_back(vu);
    }
    if (pos.size() > 4) { sym.ncorr = -1; return false; }
    sym.ncorr = (int32_t)pos.size();
    for (size_t j = 0; j < pos.size(); j++) {
        const int vu = pos[j], u = vu & 7, v = vu >> 3;
        sym.corr_pos[j] = vu;
        for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) {
            const int yy = y < 4 ? y : 7 - y, xx = x < 4 ? x : 7 - x;
            int sg = 1; if (x >= 4 && (u & 1)) sg = -sg; if (y >= 4 && (v & 1)) sg = -sg;
            sym.corr[j][y * 8 + x] = li[(y * 8 + x) * 64 + vu] - sg * li[(yy * 8 + xx) * 64 + vu];
        }
    }
    return true;
}

int jsgpu_set_idct_tables(jsgpu_ctx* ctx, const int32_t* li, const float* lf)
{
    if (!ctx || !li || !lf) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    IdctSym* sym = new IdctSym;
    ctx->sym_ok = build_idct_sym(li, *sym);
    ctx->baked_ok = js_idct_baked_matches(li) != 0;
    ctx->bakedf_ok = js_idctf_baked_matches(lf) != 0;
    ctx->h_li.assign(li, li + 64 * 64); ctx->h_lf.assign(lf, lf + 64 * 64);
    {   // the integer tile kernel takes its table as immediates when the baked copy matches, else from shared memory;
        // JSGPU_IDCT_TABLE=0 forces the shared-memory table (tests)
        const char* e = getenv("JSGPU_IDCT_TABLE");
        ctx->tab_baked = ctx->baked_ok && !(e && atoi(e) == 0);
    }
    cudaError_t e1 = ctx->d_li.reserve(64 * 64 * 4), e2 = ctx->d_lf.reserve(64 * 64 * 4), e3 = ctx->d_sym.reserve(sizeof(IdctSym));
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) { delete sym; return fail(ctx, JSGPU_ENOMEM, "idct table allocation failed"); }
    cudaMemcpyAsync(ctx->d_li.p, li, 64 * 64 * 4, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemcpyAsync(ctx->d_lf.p, lf, 64 * 64 * 4, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemcpyAsync(ctx->d_sym.p, sym, sizeof(IdctSym), cudaMemcpyHostToDevice, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    delete sym;
    if (e != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "idct table upload failed: %s", cudaGetErrorString(e));
    if (!ctx->have_ctab) {      // colour tables: built and verified on the device once per context
        if (ctx->d_ctab.reserve(sizeof(ColorTabs)) != cudaSuccess) return fail(ctx, JSGPU_ENOMEM, "colour table allocation failed");
        js_launch_build_color_tables((ColorTabs*)ctx->d_ctab.p, ctx->stream);
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "colour table build failed");
        ctx->have_ctab = true;
    }
    ctx->have_idct = true;
    return JSGPU_OK;
}

int jsgpu_set_options(jsgpu_ctx* ctx, const jsgpu_options* opt)
{
    if (!ctx || !opt) return JSGPU_EINVAL;
    if (opt->idct_mode < 0 || opt->idct_mode > 1) return fail(ctx, JSGPU_EINVAL, "idct_mode must be 0 (integer) or 1 (float)");
    ctx->opt = *opt;
    return JSGPU_OK;
}
int jsgpu_set_scan_error_state(jsgpu_ctx* ctx, uint32_t warn_start, int disable)
{
    if (!ctx) return JSGPU_EINVAL;
    ctx->scan_warn_start = warn_start; ctx->scan_errors_disable = disable != 0;
    return JSGPU_OK;
}
int jsgpu_get_options(jsgpu_ctx* ctx, jsgpu_options* opt) { if (!ctx || !opt) return JSGPU_EINVAL; *opt = ctx->opt; return JSGPU_OK; }

int jsgpu_upload_tables(jsgpu_ctx* ctx, const jsgpu_tables* sets, uint32_t nsets)
{
    if (!ctx || !sets || nsets == 0) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    std::vector<DevTableSet> h(nsets);
    for (uint32_t i = 0; i < nsets; i++) build_table_set(sets[i], h[i]);
    ctx->h_sets.assign(sets, sets + nsets);
    CK(ctx->d_tables.reserve(sizeof(DevTableSet) * (size_t)nsets));
    CK(cudaMemcpyAsync(ctx->d_tables.p, h.data(), sizeof(DevTableSet) * (size_t)nsets, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->set_l2.assign(nsets, {});
    for (uint32_t i = 0; i < nsets; i++) for (int k = 0; k < JS_NSLOT; k++) ctx->set_l2[i][k] = h[i].lut2_overflow[k] ? 0xffffffffu : h[i].lut2_used[k];
    ctx->nsets = nsets;
    return JSGPU_OK;
}

// ncclBroadcast(sendbuff, recvbuff, count, ncclChar = 0, root, comm, stream), resolved at run time
typedef int (*js_nccl_bcast_fn)(const void*, void*, size_t, int, int, void*, cudaStream_t);
static js_nccl_bcast_fn js_nccl_broadcast()
{
    static js_nccl_bcast_fn fn = nullptr; static bool tried = false;
    if (!tried) {
        tried = true;
        const char* names[] = { getenv("JSGPU_NCCL_LIB"), "libnccl.so.2", "libnccl.so" };
        for (const char* nm : names) {
            if (!nm) continue;
            void* h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (h) { fn = (js_nccl_bcast_fn)dlsym(h, "ncclBroadcast"); if (fn) break; }
        }
    }
    return fn;
}

int jsgpu_bcast_tables(jsgpu_ctx* ctx, jsgpu_tables* sets, uint32_t nsets, void* nccl_comm, int root)
{
    if (!ctx || !sets || nsets == 0 || !nccl_comm || root < 0) return JSGPU_EINVAL;
    js_nccl_bcast_fn bcast = js_nccl_broadcast();
    if (!bcast) return fail(ctx, JSGPU_EUNSUP, "libnccl not found (set JSGPU_NCCL_LIB to its path)");
    cudaSetDevice(ctx->device);
    const size_t bytes = sizeof(jsgpu_tables) * (size_t)nsets;
    DevBuf tmp;
    CK(tmp.reserve(bytes));
    cudaError_t e = cudaMemcpyAsync(tmp.p, sets, bytes, cudaMemcpyHostToDevice, ctx->stream);     // only root's content matters
    int nr = 0;
    if (e == cudaSuccess) nr = bcast(tmp.p, tmp.p, bytes, 0 /* ncclChar */, root, nccl_comm, ctx->stream);
    if (e == cudaSuccess && nr == 0) e = cudaMemcpyAsync(sets, tmp.p, bytes, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && nr == 0) e = cudaStreamSynchronize(ctx->stream);
    if (nr != 0) return fail(ctx, JSGPU_ECUDA, "ncclBroadcast failed (ncclResult %d)", nr);
    if (e != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "table broadcast failed: %s", cudaGetErrorString(e));
    return JSGPU_OK;
}

static inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }

// Geometry + validation for one image: ImgDecode.cpp:2755-2872, 3029-3123.  Returns false when the
// reference's DecodeScanImg would return before decoding.
static bool plan_image(const jsgpu_image_desc& d, uint32_t nsets, DevImage& im)
{
    memset(&im, 0, sizeof im);
    uint32_t ns = d.num_sos_comps;
    if (ns != 1 && ns != 3) return false;                                  // :2764-2770
    if (d.num_sof_comps != 1 && d.num_sof_comps != 3) return false;        // :3029-3035
    if (d.table_set >= nsets) return false;
    uint32_t H[3], V[3];
    for (uint32_t c = 0; c < ns; c++) { H[c] = d.samp_h[c]; V[c] = d.samp_v[c]; }
    uint32_t hmax = 0, vmax = 0;
    for (uint32_t c = 0; c < ns; c++) { hmax = std::max(hmax, H[c]); vmax = std::max(vmax, V[c]); }
    if (ns == 1) { H[0] = V[0] = 1; hmax = vmax = 1; }                     // :2805-2817
    if (hmax == 0 || vmax == 0 || hmax > 4 || vmax > 4) return false;      // :2821-2825
    for (uint32_t c = 0; c < ns; c++) if (H[c] == 0 || V[c] == 0) return false;
    for (uint32_t c = 0; c < ns; c++) if (d.dqt_sel[c] > 3 || d.dht_dc_sel[c] > 3 || d.dht_ac_sel[c] > 3) return false;
    im.ns = ns; im.precision = d.precision;
    im.mcu_w = hmax * 8; im.mcu_h = vmax * 8;
    im.mcu_xmax = d.dim_x / im.mcu_w + ((d.dim_x % im.mcu_w) ? 1 : 0);
    im.mcu_ymax = d.dim_y / im.mcu_h + ((d.dim_y % im.mcu_h) ? 1 : 0);
    im.blk_xmax = im.mcu_xmax * hmax; im.blk_ymax = im.mcu_ymax * vmax;
    if (im.blk_xmax == 0 || im.blk_ymax == 0) return false;                // :2866-2868
    im.wp = im.mcu_xmax * im.mcu_w; im.hp = im.mcu_ymax * im.mcu_h;
    im.nmcu = im.mcu_xmax * im.mcu_ymax;
    im.bpm = 0;
    for (uint32_t c = 0; c < ns; c++) {
        im.H[c] = H[c]; im.V[c] = V[c];
        im.eh[c] = hmax / H[c]; im.ev[c] = vmax / V[c];                    // :2836-2839
        if (im.eh[c] == 0 || im.ev[c] == 0) return false;
        im.cw[c] = im.mcu_xmax * H[c]; im.ch[c] = im.mcu_ymax * V[c];
        im.bpm += H[c] * V[c];
        im.slot_dc[c] = d.dht_dc_sel[c]; im.slot_ac[c] = 4 + d.dht_ac_sel[c];
        im.dqt[c] = d.dqt_sel[c];
    }
    im.tab_sig = ns;
    for (uint32_t c = 0; c < ns; c++) im.tab_sig = (im.tab_sig << 6) | (im.slot_dc[c] & 3) << 4 | (im.slot_ac[c] & 3) << 2 | (im.dqt[c] & 3);
    im.restart_en = (d.restart_en && d.restart_interval) ? 1 : 0;
    im.ri = im.restart_en ? d.restart_interval : im.nmcu;
    im.nseg = (im.nmcu + im.ri - 1) / im.ri;
    im.table_set = d.table_set; im.file_pos = d.file_pos;
    im.scan_off = d.scan_offset; im.scan_len = d.scan_length;
    // fused IDCT kernel preconditions: component 1 carries the maximum sampling, chroma components
    // are identical and either fully sampled or 1 in each direction, Hmax is a power of two
    bool stdl = (H[0] == hmax && V[0] == vmax) && (hmax == 1 || hmax == 2 || hmax == 4);
    if (ns == 3) stdl = stdl && H[1] == H[2] && V[1] == V[2] && (H[1] == 1 || H[1] == hmax) && (V[1] == 1 || V[1] == vmax);
    im.tile_mcus = 32 / hmax;
    // the fused kernel double-buffers a tile's sample planes in <= 48 KB of shared memory: layouts with more than 192
    // blocks per tile (three components at 4x4, 2x4 ...) take the simple kernels like the other exotic layouts
    if (stdl && (uint64_t)im.bpm * im.tile_mcus * 128u * 2u > 48u * 1024u) stdl = false;
    im.std_layout = stdl ? 1 : 0;
    // long restart intervals (no DRI, or a DRI of an MCU row and more): the self-synchronising Huffman passes apply
    im.psync = ((uint64_t)im.ri * im.bpm >= JS_PSYNC_MIN_BLOCKS) ? 1 : 0;
    im.tiles_per_row = (im.mcu_xmax + im.tile_mcus - 1) / im.tile_mcus;
    im.valid = 1;
    return true;
}

// The plan of a batch: validation, every image's geometry and pool offsets, the work lists, the IDCT tiles, the marker-scan
// chunks and the totals, on the host.  Images plan_image refuses are skipped: status 0x80000000, no pool space.
static int plan_batch(const jsgpu_image_desc* imgs, uint32_t n, uint32_t nsets, uint64_t bitstream_bytes, BatchPlan& p, std::string& err)
{
    p = BatchPlan();
    p.img.assign(n, DevImage());
    p.layout.assign(n, jsgpu_image_layout());
    p.bits_len = bitstream_bytes;
    std::vector<uint2> items_np, litems_np, vitems;
    std::vector<uint4> tcls[3];
    for (uint32_t i = 0; i < n; i++) {
        DevImage& im = p.img[i];
        jsgpu_image_layout& lo = p.layout[i];
        bool ok = plan_image(imgs[i], nsets, im);
        if (ok && (imgs[i].scan_offset > bitstream_bytes || imgs[i].scan_length > bitstream_bytes - imgs[i].scan_offset))
            return fail(err, JSGPU_EINVAL, "image %u: scan [%llu,+%llu) outside the %llu-byte bitstream", i,
                        (unsigned long long)imgs[i].scan_offset, (unsigned long long)imgs[i].scan_length, (unsigned long long)bitstream_bytes);
        if (ok && imgs[i].scan_length >= 0x1ffffff0ull) return fail(err, JSGPU_EINVAL, "image %u: scan longer than 512 MiB (bit positions are 32-bit)", i);
        if (ok && (imgs[i].scan_offset & 15)) return fail(err, JSGPU_EINVAL, "image %u: scan_offset %llu is not 16-byte aligned (jsgpu_image_desc)", i, (unsigned long long)imgs[i].scan_offset);
        if (!ok) {            // skipped image: no pool space, but keep seg_first monotone (k_finalize_mcumap binary-searches it)
            im.valid = 0; im.nseg = 0; im.seg_first = p.nseg; lo.status = 0x80000000u; continue;
        }
        im.pix_off = p.pix; im.dib_off = p.dib; im.blk_off = p.blk; im.mcu_off = p.mcu; im.seg_first = p.nseg;
        for (uint32_t c = 0; c < im.ns; c++) { im.coef_row[c] = p.coef_rows; p.coef_rows += (uint64_t)im.cw[c] * im.ch[c]; }
        uint64_t npx = (uint64_t)im.wp * im.hp;
        im.row_off = p.rows; p.rows += im.hp; p.max_hp = std::max(p.max_hp, im.hp);
        im.mc_first = p.mc_img.size(); im.mc_n = (uint32_t)((im.scan_len + 4095) >> 12); if (im.mc_n == 0) im.mc_n = 1;
        p.mc_img.insert(p.mc_img.end(), im.mc_n, i);
        p.pix += align_up(npx, 64); p.dib += align_up(npx * 4, 256); p.blk += align_up((uint64_t)im.blk_xmax * im.blk_ymax, 64);
        p.mcu += align_up(im.nmcu, 32); p.nseg += im.nseg;
        p.max_scan_len = std::max(p.max_scan_len, im.scan_len);
        for (uint32_t k = 0; k < im.nseg; k += JS_HUFF_WARPS) p.items.push_back(make_uint2(i, k));
        for (uint32_t k = 0; k < im.nseg; k += JS_LANE_SEGS) p.litems.push_back(make_uint2(i, k));
        const uint64_t uregion = align_up(im.scan_len + (uint64_t)JS_USLACK * im.nseg + 128, 256);
        im.ubits_off = p.ubits; p.ubits += uregion;
        if (im.psync) {           // slots of the self-synchronising passes + row table of k_unstuff
            p.n_psync++;
            im.ph_nslots = (uint32_t)(uregion >> 9) + im.nseg + 2; im.ph_first = p.ph; p.ph += (uint64_t)im.ph_nslots + 1;
            im.rt_off = p.rt; p.rt += (im.scan_len >> 7) + 2ull * im.nseg + 4;
            im.cs_nslots = (uint32_t)(im.scan_len >> 12) + 2 * im.nseg + 2; im.cs_first = p.cs; p.cs += im.cs_nslots; p.max_cs = std::max(p.max_cs, im.cs_nslots);
            for (uint32_t k = 0; k < im.ph_nslots; k += JS_LANE_SEGS) vitems.push_back(make_uint2(i, k));
        } else {
            p.nseg_np += im.nseg;
            for (uint32_t k = 0; k < im.nseg; k += JS_HUFF_WARPS) items_np.push_back(make_uint2(i, k));
            for (uint32_t k = 0; k < im.nseg; k += JS_LANE_SEGS) litems_np.push_back(make_uint2(i, k));
        }
        if (im.std_layout) {
            p.n_std++;
            const uint32_t ehc = (im.ns == 3) ? im.eh[1] : 1, cls = (ehc == 1) ? 0 : (ehc == 2) ? 1 : 2;
            for (uint32_t r = 0; r < im.mcu_ymax; r++) for (uint32_t t = 0; t < im.tiles_per_row; t++) {
                uint32_t c0 = t * im.tile_mcus;
                tcls[cls].push_back(make_uint4(i, r, c0, std::min(im.tile_mcus, im.mcu_xmax - c0)));
            }
            uint32_t bpt = 0; for (uint32_t c = 0; c < im.ns; c++) bpt += im.H[c] * im.V[c] * im.tile_mcus;
            p.plane_bytes = std::max(p.plane_bytes, bpt * 128);
        } else p.n_nonstd++;
        lo.mcu_w = im.mcu_w; lo.mcu_h = im.mcu_h; lo.mcu_xmax = im.mcu_xmax; lo.mcu_ymax = im.mcu_ymax;
        lo.blk_xmax = im.blk_xmax; lo.blk_ymax = im.blk_ymax; lo.img_x = im.wp; lo.img_y = im.hp;
        lo.num_segments = im.nseg; lo.pix_off = im.pix_off; lo.dib_off = im.dib_off; lo.blk_off = im.blk_off; lo.mcu_off = im.mcu_off;
    }
    p.histo = (uint64_t)n * JSGPU_HISTO_WORDS; p.stats = (uint64_t)n * JSGPU_STAT_WORDS;
    p.n_items = (uint32_t)p.items.size(); p.n_items_np = (uint32_t)items_np.size();
    p.items.insert(p.items.end(), items_np.begin(), items_np.end());
    p.n_litems = (uint32_t)p.litems.size(); p.n_litems_np = (uint32_t)litems_np.size(); p.n_vitems = (uint32_t)vitems.size();
    p.litems.insert(p.litems.end(), litems_np.begin(), litems_np.end());
    p.litems.insert(p.litems.end(), vitems.begin(), vitems.end());
    for (int k = 0; k < 3; k++) { p.tcls_first[k] = (uint32_t)p.tiles.size(); p.tcls_count[k] = (uint32_t)tcls[k].size(); p.tiles.insert(p.tiles.end(), tcls[k].begin(), tcls[k].end()); }
    return JSGPU_OK;
}

// A new batch: the context holds none until its plan (and, for jsgpu_batch_begin, its pools) is complete
static int begin_plan(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n, uint64_t bitstream_bytes)
{
    if (!ctx->have_idct) return fail(ctx, JSGPU_ESTATE, "jsgpu_set_idct_tables() has not been called");
    if (ctx->nsets == 0) return fail(ctx, JSGPU_ESTATE, "jsgpu_upload_tables() has not been called");
    cudaSetDevice(ctx->device);
    ctx->state = JS_NO_BATCH;
    return plan_batch(imgs, n, ctx->nsets, bitstream_bytes, ctx->plan, ctx->err);
}

int jsgpu_batch_begin(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n, uint64_t bitstream_bytes)
{
    if (!ctx || !imgs || n == 0) return JSGPU_EINVAL;
    const int r = begin_plan(ctx, imgs, n, bitstream_bytes); if (r) return r;
    const BatchPlan& p = ctx->plan;
    DevBatch& b = ctx->batch;
    memset(&b, 0, sizeof b);
    // allocate; carve() sizes the sub-allocated pools from their layouts and binds them
    CK(ctx->d_img.reserve(sizeof(DevImage) * (size_t)n));
    CK(ctx->d_items.reserve(sizeof(uint2) * std::max<size_t>(p.items.size(), 1)));
    CK(ctx->d_bits.reserve(bitstream_bytes + 64));
    CK(ctx->d_ubits.reserve(p.ubits + 16384));     // + slack: a reader of corrupt data stops at the next MCU boundary, at most one MCU (<= 12 KB of bits) past the end
    CK(ctx->d_litems.reserve(sizeof(uint2) * std::max<size_t>(p.litems.size(), 1)));
    auto ph = [&](Carve& c) {       // slot arrays, 16-byte members first; two list lengths per image
        c.take(b.ph_cnt, p.ph); c.take(b.ph_aux, p.ph); c.take(b.ph_pre, p.ph); c.take(b.ph_x, p.ph);
        c.take(b.ph_ver, p.ph); c.take(b.ph_k, p.ph); c.take(b.ph_list[0], p.ph); c.take(b.ph_list[1], p.ph);
        c.take(b.ph_nl[0], n); c.take(b.ph_nl[1], n); c.skip(256);
    };
    CK(carve(ctx->d_ph, ph));
    auto rowtab = [&](Carve& c) {   // per 128-byte raw row: row mask, unstuffed bytes before it; per 4 KB chunk: three words
        c.take(b.rowmask, p.rt); c.take(b.rowtab, p.rt); c.take(b.cs_cnt, p.cs); c.take(b.cs_off, p.cs); c.take(b.cs_seg, p.cs); c.skip(256);
    };
    CK(carve(ctx->d_rowtab, rowtab));
    CK(ctx->d_tiles.reserve(sizeof(uint4) * std::max<size_t>(p.tiles.size(), 1)));
    CK(ctx->d_seg64.reserve(8 * (size_t)p.nseg + 16));
    auto seg = [&](Carve& c) {
        c.take(b.seg_start, p.nseg); c.take(b.seg_end, p.nseg); c.take(b.seg_endbits, p.nseg); c.take(b.seg_status, p.nseg);
        c.take(b.seg_ulen, p.nseg); c.take(b.scan_end, n); c.take(b.nseg_found, n); c.take(b.seg_nstuff, p.nseg);
        c.take(b.seg_stuff, (uint64_t)JS_STUFF_LIST * p.nseg); c.take(b.ovf_list, p.nseg); c.skip(64);
    };
    CK(carve(ctx->d_seg, seg));
    CK(ctx->d_coef.reserve(p.coef_rows * 128 + 4096));    // + 4096 spare bytes: no kernel addresses them (every row index is bounded by
                                                           // its plane); kept so that the pool sizes stay as measured
    CK(ctx->d_mcubits.reserve(p.mcu * 4 + 16));
    auto pix = [&](Carve& c) { c.take(b.pix_y, p.pix); c.take(b.pix_cb, p.pix); c.take(b.pix_cr, p.pix); c.skip(64); };
    CK(carve(ctx->d_pix, pix));
    CK(ctx->d_dib.reserve(p.dib + 64));
    auto blk = [&](Carve& c) { c.take(b.blk_y, p.blk); c.take(b.blk_cb, p.blk); c.take(b.blk_cr, p.blk); c.skip(64); };
    CK(carve(ctx->d_blk, blk));
    CK(ctx->d_mcumap.reserve(p.mcu * 4 + 16));
    CK(ctx->d_histo.reserve(p.histo * 4));
    CK(ctx->d_stats.reserve(p.stats * 4));
    static_assert(1 + PH_MAX_ROUNDS + 2 <= 16, "ovf_count and ph_nchg share one 64-byte block");
    auto misc = [&](Carve& c) {     // per image: brightest-pixel key, luma sum, status word; the counters; per image: exact-path flag
        c.take(b.bright_key, n); c.take(b.sum_y, n); c.take(b.img_status, n);
        c.take(b.ovf_count, 1); c.take(b.ph_nchg, 15); c.take(b.ex_flag, n); c.skip(64);
    };
    CK(carve(ctx->d_misc, misc));
    CK(ctx->d_ex.reserve((size_t)n * sizeof(JsExResult)));
    auto mc = [&](Carve& c) { c.take(b.mc_img, p.mc_img.size()); c.align(64); c.take(b.mc_state, p.mc_img.size() + 2); };
    CK(carve(ctx->d_mc, mc));
    ctx->pv_done = false;
    if (!p.mc_img.empty()) CK(cudaMemcpyAsync(b.mc_img, p.mc_img.data(), p.mc_img.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_img.p, p.img.data(), sizeof(DevImage) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    if (!p.items.empty()) CK(cudaMemcpyAsync(ctx->d_items.p, p.items.data(), sizeof(uint2) * p.items.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (!p.litems.empty()) CK(cudaMemcpyAsync(ctx->d_litems.p, p.litems.data(), sizeof(uint2) * p.litems.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (!p.tiles.empty()) CK(cudaMemcpyAsync(ctx->d_tiles.p, p.tiles.data(), sizeof(uint4) * p.tiles.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));      // the next plan rewrites these host arrays
    b.img = (const DevImage*)ctx->d_img.p; b.tables = (const DevTableSet*)ctx->d_tables.p; b.nimg = n;
    b.bits = (const uint8_t*)ctx->d_bits.p; b.bits_len = bitstream_bytes; b.nseg_total = p.nseg;
    b.seg_uoff = (unsigned long long*)ctx->d_seg64.p; b.ubits = (uint8_t*)ctx->d_ubits.p;
    b.litems = (const uint2*)ctx->d_litems.p; b.nlitems = p.n_litems;
    b.litems_np = b.litems + p.n_litems; b.nlitems_np = p.n_litems_np;
    b.vitems = b.litems_np + p.n_litems_np; b.nvitems = p.n_vitems;
    b.items = (const uint2*)ctx->d_items.p; b.nitems = p.n_items;
    b.items_np = b.items + p.n_items; b.nitems_np = p.n_items_np;
    b.tiles = (const uint4*)ctx->d_tiles.p; b.ntiles = (uint32_t)p.tiles.size(); b.tile_plane_bytes = p.plane_bytes;
    for (int k = 0; k < 3; k++) { b.tcls_first[k] = p.tcls_first[k]; b.tcls_count[k] = p.tcls_count[k]; }
    b.coef = (int16_t*)ctx->d_coef.p; b.mcu_bitpos = (uint32_t*)ctx->d_mcubits.p;
    b.dib = (uint8_t*)ctx->d_dib.p; b.mcu_map = (uint32_t*)ctx->d_mcumap.p;
    b.histo = (uint32_t*)ctx->d_histo.p; b.stats = (int32_t*)ctx->d_stats.p;
    b.mc_total = (uint32_t)p.mc_img.size(); b.ex_res = (JsExResult*)ctx->d_ex.p;
    ctx->state = JS_PLANNED;
    return JSGPU_OK;
}

int jsgpu_batch_layout(jsgpu_ctx* ctx, jsgpu_image_layout* out, uint32_t n)
{
    if (!ctx || !out) return JSGPU_EINVAL;
    if (ctx->state == JS_NO_BATCH) return fail(ctx, JSGPU_ESTATE, "no batch planned");
    std::vector<jsgpu_image_layout>& layout = ctx->plan.layout;
    if (n > layout.size()) n = (uint32_t)layout.size();
    if (ctx->state == JS_DECODED) {
        cudaSetDevice(ctx->device);
        std::vector<uint32_t> st(layout.size());
        CK(cudaMemcpyAsync(st.data(), ctx->batch.img_status, st.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        std::vector<uint32_t> ex(layout.size());
        CK(cudaMemcpyAsync(ex.data(), ctx->batch.ex_flag, ex.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        for (size_t i = 0; i < st.size(); i++) if (ctx->plan.img[i].valid) layout[i].status = st[i] | (ex[i] ? JSGPU_ST_EXACT : 0u);
    }
    memcpy(out, layout.data(), sizeof(jsgpu_image_layout) * n);
    return JSGPU_OK;
}

int jsgpu_batch_pools(jsgpu_ctx* ctx, jsgpu_pools* out)
{
    if (!ctx || !out) return JSGPU_EINVAL;
    if (ctx->state < JS_PLANNED) return fail(ctx, JSGPU_ESTATE, "%s", ctx->state == JS_LAYOUT_ONLY ? HOST_DELIVERED : "no batch planned");
    for (const JsOutput& o : js_outputs) set_ptr(out, o.host, get_ptr(&ctx->batch, o.dev));
    out->coef = ctx->batch.coef; out->bitstream = (uint8_t*)ctx->d_bits.p;
    return JSGPU_OK;
}

int jsgpu_batch_upload(jsgpu_ctx* ctx, const uint8_t* host, uint64_t bytes)
{
    if (!ctx || !host) return JSGPU_EINVAL;
    if (ctx->state < JS_PLANNED) return fail(ctx, JSGPU_ESTATE, "no batch planned");
    if (bytes > ctx->plan.bits_len) return fail(ctx, JSGPU_EINVAL, "upload larger than the planned bitstream");
    cudaSetDevice(ctx->device);
    CK(cudaMemcpyAsync(ctx->d_bits.p, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return JSGPU_OK;
}

// The detailed decode of this batch's image ctx->dtl.image (jsgpu_set_detail): picks the path and sizes the event and matrix
// arrays.  A healthy image (status 0 after the Huffman stage: one sync) is decoded one thread per MCU; the count pass and scan
// run now (a second sync reads the totals, so the arrays are sized exactly), the emit pass after the MCU file map.  Otherwise
// the serial walk fills arrays sized for the most it can report: 1 + 66 events per block (a separator per MCU; per block a
// heading, at most 64 symbols, a matrix) and one matrix per block, for the printed MCUs.
static int detail_prepare(jsgpu_ctx* ctx, const JsErrCfg& cfg, int* launches)
{
    static const bool force_walk = [] { const char* e = getenv("JSGPU_DETAIL_WALK"); return e && atoi(e) == 1; }();
    const DevBatch& b = ctx->batch;
    cudaStream_t s = ctx->stream;
    const jsgpu_detail& dtl = ctx->dtl;
    const DevImage& im = ctx->plan.img[dtl.image];
    // the walk decodes MCUs 0 .. end-1 and prints those from base on (its arithmetic: a 32-bit base, a 64-bit end)
    const uint32_t base = dtl.mcu_y * im.mcu_xmax + dtl.mcu_x;
    const uint32_t end = im.valid ? (uint32_t)std::min<unsigned long long>(im.nmcu, (unsigned long long)base + dtl.len) : 0u;
    JsDetailRange r;
    r.image = dtl.image; r.base = base; r.nprint = (base < end) ? end - base : 0u;
    r.first = (base < end) ? (base ? base - 1 : 0u) : (end ? end - 1 : 0u);
    r.n = end ? end - r.first : 0u;
    uint32_t status = 1;
    if (im.valid && !force_walk && ctx->opt.want_mcu_map) {
        CK(cudaMemcpyAsync(&status, b.img_status + dtl.image, 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    CK(ctx->d_dt_scratch.reserve((16 + JSGPU_HISTO_WORDS + 2 * (size_t)r.n) * 4));
    uint32_t* hdr = (uint32_t*)ctx->d_dt_scratch.p;
    CK(cudaMemsetAsync(hdr, 0, 16 * 4, s));
    uint64_t nev, nmat;
    if (status == 0) {
        *launches += js_launch_detail_count(b, r, hdr + 16 + JSGPU_HISTO_WORDS, hdr, cfg, s);
        uint32_t tot[2];
        CK(cudaMemcpyAsync(tot, hdr, sizeof tot, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        nev = tot[0]; nmat = tot[1];
    } else {
        nev = (uint64_t)r.nprint * (1 + (uint64_t)im.bpm * 66);
        nmat = (uint64_t)r.nprint * im.bpm;
    }
    CK(ctx->d_dt_ev.reserve(std::max<uint64_t>(nev, 1) * sizeof(jsgpu_detail_event)));
    CK(ctx->d_dt_mat.reserve(std::max<uint64_t>(nmat, 1) * 64 * sizeof(int16_t)));
    ctx->dt_out.ev = (jsgpu_detail_event*)ctx->d_dt_ev.p; ctx->dt_out.mat = (int16_t*)ctx->d_dt_mat.p; ctx->dt_out.hdr = hdr;
    ctx->dt_out.ev_cap = nev; ctx->dt_out.mat_cap = nmat;
    ctx->dt_range = r;
    ctx->dt_parallel = status == 0;
    return JSGPU_OK;
}

int jsgpu_batch_decode(jsgpu_ctx* ctx)
{
    if (!ctx) return JSGPU_EINVAL;
    if (ctx->state < JS_PLANNED) return fail(ctx, JSGPU_ESTATE, "no batch planned (the last jsgpu_decode_batch_host left only its layout here)");
    cudaSetDevice(ctx->device);
    DevBatch& b = ctx->batch; const BatchPlan& p = ctx->plan;
    b.decode_ac = ctx->opt.decode_ac; b.want_histo = ctx->opt.want_histo; b.idct_mode = ctx->opt.idct_mode;
    b.any_p12 = 0; for (const DevImage& im : p.img) if (im.valid && im.precision > 8) b.any_p12 = 1;
    b.lane_nlut = 1; b.lane_l2_smem = 1; b.max_nseg = 0;
    for (const DevImage& im : p.img) if (im.valid) b.max_nseg = std::max(b.max_nseg, im.nseg);
    for (const DevImage& im : p.img) if (im.valid) {
        uint32_t seen = 0, nl = 0;
        for (uint32_t c = 0; c < im.ns; c++) for (int cls = 0; cls < 2; cls++) {
            const uint32_t slot = cls ? im.slot_ac[c] : im.slot_dc[c];
            if (!(seen >> slot & 1)) { seen |= 1u << slot; nl++; if (ctx->set_l2[im.table_set][slot] > JS_LANE_L2S) b.lane_l2_smem = 0; }
        }
        b.lane_nlut = std::max(b.lane_nlut, nl);
    }
    cudaStream_t s = ctx->stream;
    int launches = 0;
    CK(cudaEventRecord(ctx->ev[0], s));
    // clear accumulators (the reference memsets its maps: ImgDecode.cpp:2900,2924-2928,2965)
    CK(cudaMemsetAsync(b.histo, 0, p.histo * 4, s));
    CK(cudaMemsetAsync(b.stats, 0, p.stats * 4, s));
    CK(cudaMemsetAsync(b.bright_key, 0, (size_t)b.nimg * (8 + 8 + 4) + 4, s));      // + ovf_count
    CK(cudaMemsetAsync(b.mcu_map, 0, p.mcu * 4, s));
    CK(cudaMemsetAsync(b.blk_y, 0, p.blk * 2 * 3, s));
    // exotic sampling layouts leave pixels of a component unwritten (a component with 1 < H < Hmax covers only part of the MCU): they
    // read as the 0 the reference's memset left there (ImgDecode.cpp:2924-2928); standard layouts write every pixel
    if (p.n_nonstd) CK(cudaMemsetAsync(b.pix_y, 0, p.pix * 2 * 3, s));
    launches += js_launch_marker_scan(b, p.max_scan_len, s);
    // long intervals: chunk-parallel unstuffing into the pre-zeroed pool (chunk edges are OR-ed in)
    if (p.n_psync) CK(cudaMemsetAsync(ctx->d_ubits.p, 0, p.ubits + 16384, s));
    if (p.n_psync < p.n_std + p.n_nonstd) launches += js_launch_unstuff(b, s);
    if (p.n_psync) launches += js_launch_unstuff_long(b, p.max_cs, s);
    CK(cudaEventRecord(ctx->ev[1], s));
    {
        // huff_kernel: 1 = one warp per restart interval for everything, 2 = one lane per restart interval for everything,
        // 0/3 = images with long intervals (no DRI ...) through the self-synchronising passes + the lane kernel over their
        // virtual intervals, the others through the lane kernel when there are many intervals, else the warp kernel
        int hk = ctx->opt.huff_kernel;
        const bool selfsync = (hk == 0 || hk == 3) && b.nvitems > 0 && b.lane_l2_smem;
        DevBatch bh = b;
        uint32_t nseg_short = b.nseg_total;
        if (selfsync) { bh.items = b.items_np; bh.nitems = b.nitems_np; bh.litems = b.litems_np; bh.nlitems = b.nlitems_np; nseg_short = p.nseg_np; }
        else bh.nvitems = 0;
        if (hk == 0 || hk == 3) hk = (nseg_short >= 4096) ? 2 : 1;       // many short intervals -> lane kernel
        if (hk == 2) launches += js_launch_huffman_lane(bh, ctx->sm_count, s);
        else launches += js_launch_huffman_warp(bh, ctx->sm_count, s);
        if (selfsync) {
            launches += js_launch_selfsync(bh, ctx->sm_count, s);
            launches += js_launch_huffman_lane_vseg(bh, ctx->sm_count, s);
        }
        // the detailed decode of a healthy image: count pass and scan here, events after the MCU file map (below)
        ctx->ex_cfg = JsErrCfg{ctx->opt.scan_err_max, ctx->scan_warn_start, ctx->scan_errors_disable ? 1u : 0u};
        ctx->dt_done = ctx->dt_parallel = false;
        jsgpu_detail dtl = ctx->dtl;
        if (dtl.enable && dtl.image < b.nimg) {
            int rc = detail_prepare(ctx, ctx->ex_cfg, &launches);
            if (rc != JSGPU_OK) return rc;
            ctx->dt_done = true;
            if (ctx->dt_parallel) dtl.enable = 0;
        } else dtl.enable = 0;
        // damaged images (status word != 0) are decoded again with the reference's semantics (and the detail image, when it takes
        // the serial walk); returns at once for the others
        launches += js_launch_exact(b, ctx->ex_cfg, dtl, ctx->dt_out, ctx->dt_done ? (uint32_t*)ctx->d_dt_scratch.p + 16 : nullptr, s);
    }
    // The MCU file map depends on the Huffman stage only: its kernels run on a second stream while the IDCT kernel has the device
    // (they are short and latency-bound); the scalar statistics below wait for both.
    bool maps_forked = false;
    if (ctx->opt.want_mcu_map) {
        CK(cudaEventRecord(ctx->evx[0], s));
        CK(cudaStreamWaitEvent(ctx->stream2, ctx->evx[0], 0));
        launches += js_launch_finalize_maps(b, ctx->stream2);
        launches += js_launch_finalize_emptied(b, ctx->stream2);
        if (ctx->dt_parallel) launches += js_launch_detail_emit(b, ctx->dt_range, (const uint32_t*)ctx->d_dt_scratch.p + 16 + JSGPU_HISTO_WORDS, ctx->dt_out, ctx->stream2);
        CK(cudaEventRecord(ctx->evx[1], ctx->stream2));
        maps_forked = true;
    }
    CK(cudaEventRecord(ctx->ev[2], s));
    {
        // fused tile kernel for the images with standard sampling layouts, when the integer table decomposes (integer IDCT) or
        // the float table is the baked one, bit for bit (float IDCT, the reference's default build); everything else (exotic
        // sampling, a host table the tile kernel cannot use, idct_kernel = 1) takes the simple kernels
        const bool flt = ctx->opt.idct_mode == 1;
        const bool fused = ctx->opt.idct_kernel != 1 && b.ntiles > 0 && (flt ? ctx->bakedf_ok : ctx->sym_ok);
        if (fused)
            launches += js_launch_idct_fused(b, (const IdctSym*)ctx->d_sym.p, (const ColorTabs*)ctx->d_ctab.p, ctx->sm_count,
                                             flt ? JS_TILE_FLOAT : ctx->tab_baked ? JS_TILE_INT_BAKED : JS_TILE_INT_SMEM, s);
        if (!fused || p.n_nonstd > 0) {
            DevBatch bs = b; bs.simple_only_nonstd = fused ? 1 : 0;
            launches += js_launch_idct_simple(bs, (const int32_t*)ctx->d_li.p, (const float*)ctx->d_lf.p, s);
        }
    }
    CK(cudaEventRecord(ctx->ev[3], s));
    if (maps_forked) CK(cudaStreamWaitEvent(s, ctx->evx[1], 0));
    launches += js_launch_finalize_stats(b, s);
    // CalcChannelPreview() with non-default settings (ImgDecode.cpp:3641-3643): the DIB again, from the pixel maps
    ctx->pv_done = false;
    if (!preview_is_default(ctx->pv)) {
        int rc = run_preview(ctx, ctx->pv, &launches);
        if (rc != JSGPU_OK) return rc;
    }
    CK(cudaEventRecord(ctx->ev[4], s));
    CK(cudaGetLastError());
    ctx->launches = launches;
    ctx->state = JS_DECODED;
    return JSGPU_OK;
}

int jsgpu_set_preview(jsgpu_ctx* ctx, const jsgpu_preview* p)
{
    if (!ctx || !p) return JSGPU_EINVAL;
    if (p->mode < 0 || p->mode > 8) return fail(ctx, JSGPU_EINVAL, "preview mode must be 0..8 (snoop.h:100-108)");
    ctx->pv = *p;
    if (ctx->pv.mode == 0) ctx->pv.mode = 1;
    return JSGPU_OK;
}

int jsgpu_batch_preview(jsgpu_ctx* ctx, const jsgpu_preview* p)
{
    if (!ctx || !p) return JSGPU_EINVAL;
    if (p->mode < 0 || p->mode > 8) return fail(ctx, JSGPU_EINVAL, "preview mode must be 0..8 (snoop.h:100-108)");
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "no device-resident decode to recolour");
    cudaSetDevice(ctx->device);
    jsgpu_preview pv = *p; if (pv.mode == 0) pv.mode = 1;
    int launches = 0;
    int rc = run_preview(ctx, pv, &launches);
    if (rc != JSGPU_OK) return rc;
    CK(cudaGetLastError());
    ctx->launches = launches;
    return JSGPU_OK;
}

int jsgpu_set_detail(jsgpu_ctx* ctx, const jsgpu_detail* d)
{
    if (!ctx || !d) return JSGPU_EINVAL;
    ctx->dtl = *d;
    return JSGPU_OK;
}

int jsgpu_batch_detail_info(jsgpu_ctx* ctx, uint32_t info[4])
{
    if (!ctx || !info) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED || !ctx->dt_done) return fail(ctx, JSGPU_ESTATE, "the last decode collected no detailed decode (jsgpu_set_detail)");
    cudaSetDevice(ctx->device);
    CK(cudaMemcpyAsync(info, ctx->dt_out.hdr, 2 * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    info[2] = ctx->dt_parallel ? JSGPU_DETAIL_PARALLEL : JSGPU_DETAIL_SERIAL; info[3] = 0;
    return JSGPU_OK;
}

int jsgpu_batch_detail_events(jsgpu_ctx* ctx, uint32_t first, uint32_t n, jsgpu_detail_event* out)
{
    if (!ctx || (!out && n)) return JSGPU_EINVAL;
    uint32_t info[4];
    int rc = jsgpu_batch_detail_info(ctx, info);
    if (rc != JSGPU_OK) return rc;
    if ((uint64_t)first + n > std::min<uint64_t>(info[0], ctx->dt_out.ev_cap))
        return fail(ctx, JSGPU_EINVAL, "events %u..%llu asked, the detailed decode has %u", first, (unsigned long long)first + n, info[0]);
    if (n) CK(cudaMemcpyAsync(out, ctx->dt_out.ev + first, (size_t)n * sizeof *out, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

int jsgpu_batch_detail_matrices(jsgpu_ctx* ctx, uint32_t first, uint32_t n, int16_t* out)
{
    if (!ctx || (!out && n)) return JSGPU_EINVAL;
    uint32_t info[4];
    int rc = jsgpu_batch_detail_info(ctx, info);
    if (rc != JSGPU_OK) return rc;
    if ((uint64_t)first + n > std::min<uint64_t>(info[1], ctx->dt_out.mat_cap))
        return fail(ctx, JSGPU_EINVAL, "matrices %u..%llu asked, the detailed decode has %u", first, (unsigned long long)first + n, info[1]);
    if (n) CK(cudaMemcpyAsync(out, ctx->dt_out.mat + (size_t)first * 64, (size_t)n * 64 * sizeof *out, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

int jsgpu_batch_detail(jsgpu_ctx* ctx, jsgpu_detail_dump* out)
{
    if (!ctx || !out) return JSGPU_EINVAL;
    uint32_t info[4];
    int rc = jsgpu_batch_detail_info(ctx, info);
    if (rc != JSGPU_OK) return rc;
    memset(out, 0, sizeof *out);
    out->nevents = info[0]; out->nblocks = info[1];
    rc = jsgpu_batch_detail_events(ctx, 0, std::min<uint32_t>(info[0], JSGPU_MAX_DETAIL_EVENTS), out->ev);
    if (rc == JSGPU_OK) rc = jsgpu_batch_detail_matrices(ctx, 0, std::min<uint32_t>(info[1], JSGPU_MAX_DETAIL_BLOCKS), &out->matrix[0][0]);
    return rc;
}

int jsgpu_batch_export(jsgpu_ctx* ctx, uint32_t image, int mode, void* host_out, uint64_t bytes)
{
    if (!ctx || !host_out) return JSGPU_EINVAL;
    if (mode < JSGPU_EXPORT_RGB8 || mode > JSGPU_EXPORT_YCC8) return fail(ctx, JSGPU_EINVAL, "export mode must be 0 (RGB8), 1 (RGB16) or 2 (YCC8)");
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "no device-resident decode to export");
    if (image >= ctx->plan.img.size()) return fail(ctx, JSGPU_EINVAL, "image index out of range");
    const DevImage& im = ctx->plan.img[image];
    if (!im.valid) return fail(ctx, JSGPU_EUNSUP, "image %u was skipped", image);
    if (mode == JSGPU_EXPORT_YCC8 && im.ns != 3) return fail(ctx, JSGPU_EUNSUP, "YCC export needs a three-component scan");
    const uint64_t npx = (uint64_t)im.wp * im.hp, need = npx * (mode == JSGPU_EXPORT_RGB16 ? 6 : 3);
    if (bytes < need) return fail(ctx, JSGPU_EINVAL, "export buffer too small: %llu < %llu bytes", (unsigned long long)bytes, (unsigned long long)need);
    cudaSetDevice(ctx->device);
    DevBuf tmp;
    CK(tmp.reserve((size_t)need + 64));
    js_launch_export(ctx->batch, image, mode, (uint8_t*)tmp.p, npx, ctx->sm_count, ctx->stream);
    cudaError_t e = cudaMemcpyAsync(host_out, tmp.p, (size_t)need, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "export failed: %s", cudaGetErrorString(e));
    return JSGPU_OK;
}

int jsgpu_batch_colour_stats(jsgpu_ctx* ctx, uint32_t image, jsgpu_colour_stats* out)
{
    if (!ctx || !out) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED || !ctx->pv_done) return fail(ctx, JSGPU_ESTATE, "no preview pass has run on this batch (jsgpu_set_preview / jsgpu_batch_preview)");
    if (image >= ctx->plan.img.size()) return fail(ctx, JSGPU_EINVAL, "image index out of range");
    cudaSetDevice(ctx->device);
    CK(cudaMemcpyAsync(out, (const jsgpu_colour_stats*)ctx->d_cstats.p + image, sizeof *out, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

int jsgpu_timer_start(jsgpu_ctx* ctx)
{
    if (!ctx) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    CK(cudaEventRecord(ctx->tev[0], ctx->stream));
    return JSGPU_OK;
}
int jsgpu_timer_stop(jsgpu_ctx* ctx, float* ms)
{
    if (!ctx || !ms) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    CK(cudaEventRecord(ctx->tev[1], ctx->stream));
    CK(cudaEventSynchronize(ctx->tev[1]));
    CK(cudaEventElapsedTime(ms, ctx->tev[0], ctx->tev[1]));
    return JSGPU_OK;
}

int jsgpu_batch_launches(jsgpu_ctx* ctx) { return ctx ? ctx->launches : JSGPU_EINVAL; }

int jsgpu_batch_errors(jsgpu_ctx* ctx, uint32_t image, jsgpu_scan_errors* out)
{
    if (!ctx || !out) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "no device-resident decode to report on");
    if (image >= ctx->plan.img.size()) return fail(ctx, JSGPU_EINVAL, "image index out of range");
    cudaSetDevice(ctx->device);
    uint32_t flag = 0;
    CK(cudaMemcpyAsync(&flag, ctx->batch.ex_flag + image, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const bool detail_walk = ctx->dt_done && ctx->dtl.enable && ctx->dtl.image == image;      // a healthy image walked for its detailed decode
    if (!flag && !detail_walk) return fail(ctx, JSGPU_ESTATE, "image %u did not take the serial error path", image);
    CK(cudaMemcpyAsync(out, ctx->batch.ex_res + image, sizeof *out, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

int jsgpu_batch_error_events(jsgpu_ctx* ctx, uint32_t image, uint32_t first, uint32_t n, jsgpu_scan_event* out)
{
    if (!ctx || (!out && n)) return JSGPU_EINVAL;
    std::unique_ptr<jsgpu_scan_errors> e(new jsgpu_scan_errors);
    int rc = jsgpu_batch_errors(ctx, image, e.get());
    if (rc != JSGPU_OK) return rc;
    const uint32_t nev = e->nevents;
    if ((uint64_t)first + n > nev) return fail(ctx, JSGPU_EINVAL, "events %u..%llu asked, image %u has %u", first, (unsigned long long)first + n, image, nev);
    if ((uint64_t)first + n <= JSGPU_MAX_EVENTS) { memcpy(out, e->ev + first, (size_t)n * sizeof *out); return JSGPU_OK; }
    // past the first JSGPU_MAX_EVENTS: walk the image again for its events alone, into a buffer sized for all of them
    const size_t hdr = sizeof(JsExResult) + JSGPU_HISTO_WORDS * 4;
    CK(ctx->d_ex_all.reserve(hdr + (size_t)nev * sizeof(JsExEvent)));
    uint8_t* base = (uint8_t*)ctx->d_ex_all.p;
    JsExEvent* ev = (JsExEvent*)(base + hdr);
    js_launch_exact_events(ctx->batch, image, ctx->ex_cfg, (JsExResult*)base, (uint32_t*)(base + sizeof(JsExResult)), ev, nev, ctx->stream);
    CK(cudaGetLastError());
    uint32_t again = 0;
    CK(cudaMemcpyAsync(&again, &((JsExResult*)base)->nevents, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(out, ev + first, (size_t)n * sizeof *out, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (again != nev) return fail(ctx, JSGPU_ECUDA, "the events-only walk of image %u found %u events, the decode %u", image, again, nev);
    return JSGPU_OK;
}

int jsgpu_batch_checksums(jsgpu_ctx* ctx, uint64_t* ck, uint32_t n)
{
    if (!ctx || !ck) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "no device-resident decode to checksum");
    if (n > ctx->plan.img.size()) n = (uint32_t)ctx->plan.img.size();
    cudaSetDevice(ctx->device);
    static_assert(JSGPU_CK_WORDS == JSGPU_CK_WORDS_INTERNAL, "checksum layout");
    DevBuf tmp;
    CK(tmp.reserve((size_t)ctx->plan.img.size() * JSGPU_CK_WORDS * 8));
    js_launch_checksums(ctx->batch, (unsigned long long*)tmp.p, ctx->stream);
    cudaError_t e = cudaMemcpyAsync(ck, tmp.p, (size_t)n * JSGPU_CK_WORDS * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "checksum kernel failed: %s", cudaGetErrorString(e));
    return JSGPU_OK;
}

int jsgpu_batch_selfsync_info(jsgpu_ctx* ctx, uint32_t* info, uint32_t n)
{
    if (!ctx || !info || n < 4) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "no device-resident decode to report on");
    cudaSetDevice(ctx->device);
    memset(info, 0, sizeof(uint32_t) * n);
    info[0] = ctx->plan.n_psync; info[1] = (uint32_t)std::min<uint64_t>(ctx->plan.ph, 0xffffffffu); info[2] = PH_MAX_ROUNDS;
    uint32_t h[PH_MAX_ROUNDS + 2] = {};
    if (ctx->plan.n_psync) {
        CK(cudaMemcpyAsync(h, ctx->batch.ph_nchg, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
    }
    for (uint32_t r = 1; r <= PH_MAX_ROUNDS && 2 + r < n; r++) info[2 + r] = h[r];
    return JSGPU_OK;
}

int jsgpu_batch_stage_ms(jsgpu_ctx* ctx, float* ms5)
{
    if (!ctx || !ms5) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "nothing decoded yet");
    cudaSetDevice(ctx->device);
    CK(cudaEventSynchronize(ctx->ev[4]));
    for (int i = 0; i < 4; i++) CK(cudaEventElapsedTime(&ms5[i], ctx->ev[i], ctx->ev[i + 1]));
    CK(cudaEventElapsedTime(&ms5[4], ctx->ev[0], ctx->ev[4]));
    return JSGPU_OK;
}

int jsgpu_batch_download(jsgpu_ctx* ctx, int which, uint32_t image, void* dst, uint64_t bytes)
{
    if (!ctx || !dst) return JSGPU_EINVAL;
    if (ctx->state != JS_DECODED) return fail(ctx, JSGPU_ESTATE, "%s", ctx->state == JS_LAYOUT_ONLY ? HOST_DELIVERED : "nothing decoded yet");
    if (image >= ctx->plan.img.size()) return fail(ctx, JSGPU_EINVAL, "image index out of range");
    cudaSetDevice(ctx->device);
    const DevImage& im = ctx->plan.img[image];
    if (!im.valid) return fail(ctx, JSGPU_EUNSUP, "image %u was not decoded", image);
    if (which < 0 || which > JSGPU_OUT_STATS) return fail(ctx, JSGPU_EINVAL, "unknown output selector %d", which);
    const JsOutput& o = js_outputs[which];
    const uint8_t* src = (const uint8_t*)get_ptr(&ctx->batch, o.dev) + out_off(o, im, image) * o.elem;
    const uint64_t avail = (o.chroma && im.ns != 3) ? 0 : o.count(im) * o.elem;
    if (bytes > avail) return fail(ctx, JSGPU_EINVAL, "output %d of image %u has %llu bytes, %llu requested", which, image,
                                   (unsigned long long)avail, (unsigned long long)bytes);
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

// One context, one stream: upload, decode, pooled D2H (each pool is one contiguous copy in batch order).
static int decode_host_single(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n, const uint8_t* bits, uint64_t bytes,
                              const jsgpu_host_outputs* out, bool wait)
{
    int r = jsgpu_batch_begin(ctx, imgs, n, bytes); if (r) return r;
    r = jsgpu_batch_upload(ctx, bits, bytes); if (r) return r;
    r = jsgpu_batch_decode(ctx); if (r) return r;
    for (const JsOutput& o : js_outputs)
        if (void* h = get_ptr(out, o.host))
            CK(cudaMemcpyAsync(h, get_ptr(&ctx->batch, o.dev), ctx->plan.*o.total * o.elem, cudaMemcpyDeviceToHost, ctx->stream));
    if (wait) CK(cudaStreamSynchronize(ctx->stream));
    return JSGPU_OK;
}

// Host bitstream in, every reference output in host buffers out.  A large batch is cut into JS_HOST_CHUNKS image ranges,
// each on its own stream with its own pools: the device-to-host copy of one range (PCIe-bound, most of the call) overlaps
// upload and decode of the next ones.  From the moment it is planned this context holds the batch layout (and, once
// decoded, the statuses) only: JS_LAYOUT_ONLY.
#define JS_HOST_CHUNKS 8u
int jsgpu_decode_batch_host(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n, const uint8_t* bits, uint64_t bytes,
                            const jsgpu_host_outputs* out)
{
    if (!ctx || !imgs || !bits || !out) return JSGPU_EINVAL;
    static const uint64_t min_bytes = getenv("JSGPU_HOST_CHUNK_MIN_BYTES") ? strtoull(getenv("JSGPU_HOST_CHUNK_MIN_BYTES"), nullptr, 10) : (64ull << 20);
    bool chunked = n >= 2 * JS_HOST_CHUNKS && bytes >= min_bytes && !ctx->h_sets.empty() && !ctx->h_li.empty();
    for (uint32_t i = 1; chunked && i < n; i++)             // chunk bitstreams must be contiguous, 16-byte aligned ranges
        if (imgs[i].scan_offset < imgs[i - 1].scan_offset + imgs[i - 1].scan_length || (imgs[i].scan_offset & 15)) chunked = false;
    if (chunked && ((imgs[0].scan_offset & 15) || imgs[n - 1].scan_offset + imgs[n - 1].scan_length > bytes)) chunked = false;
    if (!chunked) return decode_host_single(ctx, imgs, n, bits, bytes, out, true);

    // global layout (offsets of every image in the host pools) without device allocations
    int r = begin_plan(ctx, imgs, n, bytes); if (r) return r;
    ctx->state = JS_LAYOUT_ONLY;
    while (ctx->kids.size() < JS_HOST_CHUNKS) {
        jsgpu_ctx* k = nullptr;
        r = jsgpu_init(ctx->device, &k); if (r) return fail(ctx, r, "chunk context: %s", jsgpu_strerror(r));
        ctx->kids.push_back(k);
    }
    std::vector<jsgpu_image_desc> d;
    for (uint32_t c = 0; c < JS_HOST_CHUNKS; c++) {
        jsgpu_ctx* k = ctx->kids[c];
        const uint32_t i0 = (uint32_t)((uint64_t)n * c / JS_HOST_CHUNKS), i1 = (uint32_t)((uint64_t)n * (c + 1) / JS_HOST_CHUNKS);
        // (re)configure the chunk context like this one
        jsgpu_options o = ctx->opt;
        r = jsgpu_set_options(k, &o); if (r) return fail(ctx, r, "%s", k->err.c_str());
        k->scan_warn_start = ctx->scan_warn_start; k->scan_errors_disable = ctx->scan_errors_disable;
        k->pv = ctx->pv;
        if (!k->have_idct || k->h_li != ctx->h_li) { r = jsgpu_set_idct_tables(k, ctx->h_li.data(), ctx->h_lf.data()); if (r) return fail(ctx, r, "%s", k->err.c_str()); }
        if (k->h_sets.size() != ctx->h_sets.size() || memcmp(k->h_sets.data(), ctx->h_sets.data(), sizeof(jsgpu_tables) * ctx->h_sets.size()) != 0) {
            r = jsgpu_upload_tables(k, ctx->h_sets.data(), (uint32_t)ctx->h_sets.size()); if (r) return fail(ctx, r, "%s", k->err.c_str());
        }
        const uint64_t base = imgs[i0].scan_offset, end = imgs[i1 - 1].scan_offset + imgs[i1 - 1].scan_length;
        d.assign(imgs + i0, imgs + i1);
        for (auto& x : d) x.scan_offset -= base;
        uint32_t iv = i0;                                    // first image of the chunk that occupies pool space (skipped images do not)
        while (iv < i1 && !ctx->plan.img[iv].valid) iv++;
        static const DevImage none = {};
        const DevImage& f = (iv < i1) ? ctx->plan.img[iv] : none;    // its offsets in the global pools = where this chunk's outputs start
        jsgpu_host_outputs o2 = {};
        for (const JsOutput& o : js_outputs)
            if (uint8_t* h = (uint8_t*)get_ptr(out, o.host)) set_ptr(&o2, o.host, h + out_off(o, f, i0) * o.elem);
        r = decode_host_single(k, d.data(), i1 - i0, bits + base, end - base, &o2, false);
        if (r) {
            // earlier chunks still have copies in flight into the caller's buffers: let them land before handing control back
            for (uint32_t c2 = 0; c2 < c; c2++) cudaStreamSynchronize(ctx->kids[c2]->stream);
            return fail(ctx, r, "chunk %u: %s", c, k->err.c_str());
        }
    }
    ctx->launches = 0;
    for (uint32_t c = 0; c < JS_HOST_CHUNKS; c++) {
        jsgpu_ctx* k = ctx->kids[c];
        {
            const cudaError_t e = cudaStreamSynchronize(k->stream);
            if (e != cudaSuccess) {
                for (uint32_t c2 = c + 1; c2 < JS_HOST_CHUNKS; c2++) cudaStreamSynchronize(ctx->kids[c2]->stream);
                return fail(ctx, JSGPU_ECUDA, "chunk %u: %s", c, cudaGetErrorString(e));
            }
        }
        const uint32_t i0 = (uint32_t)((uint64_t)n * c / JS_HOST_CHUNKS), i1 = (uint32_t)((uint64_t)n * (c + 1) / JS_HOST_CHUNKS);
        std::vector<jsgpu_image_layout> lo(i1 - i0);
        r = jsgpu_batch_layout(k, lo.data(), i1 - i0);
        if (r) { for (uint32_t c2 = c + 1; c2 < JS_HOST_CHUNKS; c2++) cudaStreamSynchronize(ctx->kids[c2]->stream); return fail(ctx, r, "%s", k->err.c_str()); }
        for (uint32_t i = i0; i < i1; i++) ctx->plan.layout[i].status = lo[i - i0].status;
        ctx->launches += k->launches;
    }
    return JSGPU_OK;
}

int jsgpu_host_copy_rate(jsgpu_ctx* ctx, int direction, uint64_t bytes, int reps, float* gbs)
{
    if (!ctx || !gbs || bytes == 0 || reps < 1 || direction < 0 || direction > 1) return JSGPU_EINVAL;
    cudaSetDevice(ctx->device);
    void* h = nullptr; void* d = nullptr;
    if (cudaMallocHost(&h, bytes) != cudaSuccess) return fail(ctx, JSGPU_ENOMEM, "pinned allocation of %llu bytes failed", (unsigned long long)bytes);
    if (cudaMalloc(&d, bytes) != cudaSuccess) { cudaFreeHost(h); return fail(ctx, JSGPU_ENOMEM, "device allocation of %llu bytes failed", (unsigned long long)bytes); }
    memset(h, 1, bytes);                                        // touch the pages (first-touch NUMA placement happens here)
    cudaMemsetAsync(d, 0, bytes, ctx->stream);
    float best = 0.f; cudaError_t e = cudaSuccess;
    for (int r = 0; r < reps + 1 && e == cudaSuccess; r++) {     // first repetition = warm-up
        cudaEventRecord(ctx->tev[0], ctx->stream);
        e = direction ? cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, ctx->stream) : cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, ctx->stream);
        cudaEventRecord(ctx->tev[1], ctx->stream);
        if (e == cudaSuccess) e = cudaEventSynchronize(ctx->tev[1]);
        float ms = 0.f;
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, ctx->tev[0], ctx->tev[1]);
        if (r > 0 && ms > 0.f) best = std::max(best, (float)(bytes / 1e6 / ms));
    }
    cudaFree(d); cudaFreeHost(h);
    if (e != cudaSuccess) return fail(ctx, JSGPU_ECUDA, "copy-rate probe failed: %s", cudaGetErrorString(e));
    *gbs = best;
    return JSGPU_OK;
}

int jsgpu_search_bytes(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, const uint8_t* patterns, const uint32_t* lens, uint32_t npat,
                       uint64_t* counts, uint32_t* pos, uint64_t cap)
{
    if (!ctx) return JSGPU_EINVAL;
    if (!counts || !lens || !patterns || (n && !data) || (cap && !pos) || npat == 0 || npat > JSGPU_SEARCH_MAX_PATTERNS)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_search_bytes: bad arguments (npat %u, 1..%d patterns)", npat, JSGPU_SEARCH_MAX_PATTERNS);
    for (uint32_t k = 0; k < npat; k++)
        if (lens[k] < JSGPU_SEARCH_MIN_LEN || lens[k] > JSGPU_SEARCH_MAX_LEN)
            return fail(ctx, JSGPU_EINVAL, "jsgpu_search_bytes: pattern %u is %u bytes (%d..%d)", k, lens[k], JSGPU_SEARCH_MIN_LEN, JSGPU_SEARCH_MAX_LEN);
    if (n >> 32)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_search_bytes: %llu bytes: files of 2^32 bytes or more do not fit 32-bit offsets",
                    (unsigned long long)n);
    return js_search_run(&ctx->search, ctx->device, ctx->sm_count, data, n, patterns, lens, npat, counts, pos, cap, ctx->err);
}

int jsgpu_find_value(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, uint64_t start, uint32_t value, uint32_t len, int forward,
                     const jsgpu_overlay* overlays, uint32_t noverlays, int* found, uint64_t* found_pos)
{
    if (!ctx) return JSGPU_EINVAL;
    if (!found || !found_pos || (n && !data) || (noverlays && !overlays) || len < 1 || len > 4)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_value: bad arguments (len %u, 1..4)", len);
    for (uint32_t k = 0; k < noverlays; k++)
        if (overlays[k].len && !overlays[k].data) return fail(ctx, JSGPU_EINVAL, "jsgpu_find_value: overlay %u has no data", k);
    if ((n >> 32) || start >= 0xFFFFFFFFull)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_value: %llu bytes from %llu: files of 2^32 bytes or more do not fit 32-bit offsets",
                    (unsigned long long)n, (unsigned long long)start);
    return js_find_run(&ctx->search, ctx->device, ctx->sm_count, data, n, start, value, len, forward, overlays, noverlays, found,
                       found_pos, ctx->err);
}

int jsgpu_find_all(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, uint32_t value, uint32_t len, uint64_t* count, uint32_t* pos,
                   uint64_t cap)
{
    if (!ctx) return JSGPU_EINVAL;
    if (!count || (n && !data) || (cap && !pos) || len < 1 || len > 4)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_all: bad arguments (len %u, 1..4)", len);
    if (n >> 32)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_all: %llu bytes: files of 2^32 bytes or more do not fit 32-bit offsets",
                    (unsigned long long)n);
    return js_find_all_run(&ctx->search, ctx->device, ctx->sm_count, data, n, value, len, count, pos, cap, ctx->err);
}

int jsgpu_find_markers(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, const jsgpu_overlay* overlays, uint32_t noverlays,
                       uint32_t* soi_pos, uint64_t soi_cap, uint64_t* nsoi, uint32_t* term_pos, uint64_t term_cap, uint64_t* nterm)
{
    if (!ctx) return JSGPU_EINVAL;
    if (!nsoi || !nterm || (n && !data) || (noverlays && !overlays) || (soi_cap && !soi_pos) || (term_cap && !term_pos))
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_markers: bad arguments");
    for (uint32_t k = 0; k < noverlays; k++)
        if (overlays[k].len && !overlays[k].data) return fail(ctx, JSGPU_EINVAL, "jsgpu_find_markers: overlay %u has no data", k);
    if (n >> 32)
        return fail(ctx, JSGPU_EINVAL, "jsgpu_find_markers: %llu bytes: files of 2^32 bytes or more do not fit 32-bit offsets",
                    (unsigned long long)n);
    return js_find_markers_run(&ctx->search, ctx->device, ctx->sm_count, data, n, overlays, noverlays, soi_pos, soi_cap, nsoi,
                               term_pos, term_cap, nterm, ctx->err);
}

void* jsgpu_host_alloc(uint64_t bytes) { void* p = nullptr; if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr; return p; }
void  jsgpu_host_free(void* p) { if (p) cudaFreeHost(p); }

} // extern "C"
