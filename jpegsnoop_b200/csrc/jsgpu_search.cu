// jsgpu_search.cu — multi-pattern byte search (jsgpu_search_bytes, include/jsgpu.h): every position of up to 32 patterns
// (8..256 bytes) in one streaming pass, reported by the rule of JPEGsnoop's repeated CwindowBuf::BufSearchX loop
// (WindowBuf.cpp:243-331 called from JPEGsnoopDoc.cpp:1500-1512 with the next start one past the last find):
//   p is reported  <=>  the L bytes at p equal the pattern, 1 <= p <= N - 2L + 2, and p - 1 was not reported.
// The last condition makes a run of consecutive matches report every other position, from the run's first one.
//
// The file is streamed in chunks of `chunk` bytes (a multiple of the 4096-byte tile), each uploaded with its next
// maxlen - 1 bytes, from two pinned staging buffers on two streams so that the upload of chunk k+1 overlaps the search of
// chunk k.  Per chunk:
//   k_search_tiles<false>  one CTA per tile at a time stages the tile and its halo in shared memory (16-byte loads), tests
//                          every position against a 2^16-bit hash of the patterns' 8-byte prefixes (one shared-memory bit per
//                          position, whatever the number of patterns), verifies candidates byte for byte into per-pattern
//                          match bitmaps and reduces each tile to a two-state summary: the reported count and the
//                          "last position reported" flag for either value of that flag before the tile;
//   k_search_scan          one CTA per pattern chains the summaries through the chunk: every tile's incoming flag and
//                          first output index, and the chunk's count and outgoing flag;
//   k_search_tiles<true>   (second pass, only for chunks with positions inside `cap`) rewrites the tiles that report
//                          anything, in file order, into a compact per-chunk list the host copies into place.
// Device memory is two chunk buffers, the per-tile summaries and one chunk's emitted positions, whatever the file size.
// The search has its own streams and buffers: a batch resident on the same context is not touched.
// The first-match value search of Img Search Fwd / Rev (jsgpu_find_value) and the every-match value search (jsgpu_find_all),
// both at the end of the file, share them.
#include "jsgpu_internal.h"
#include <cstdlib>
#include <cstring>
#include <vector>
#include <algorithm>

#define SR_TILE     4096                 // positions per tile
#define SR_THREADS  256                  // 16 consecutive positions per thread
#define SR_HALO     272                  // bytes staged past the tile: maxlen - 1 (<= 255) and the 8-byte window, rounded to 16
#define SR_HBITS    16                   // prefix hash width
#define SR_WORDS    (SR_TILE / 32)       // match-bitmap words per pattern and tile

struct SrParams {
    uint32_t npat, maxlen;
    uint32_t len[JSGPU_SEARCH_MAX_PATTERNS];
    int64_t  maxp[JSGPU_SEARCH_MAX_PATTERNS];       // last reportable file position: N - 2L + 2 (negative: none)
    uint32_t pre_lo[JSGPU_SEARCH_MAX_PATTERNS], pre_hi[JSGPU_SEARCH_MAX_PATTERNS];   // first 8 bytes, little-endian
};
struct SrEmit {                                      // second pass: where chunk-local output index j of pattern k goes
    uint32_t lim[JSGPU_SEARCH_MAX_PATTERNS];         // ... kept only while j < lim[k] (the part that fits in `cap`)
    uint32_t base[JSGPU_SEARCH_MAX_PATTERNS];        // ... at out[base[k] + j]
};

__device__ __forceinline__ uint32_t sr_hash(uint32_t lo, uint32_t hi)
{
    return ((lo * 0x9E3779B1u) ^ (hi * 0x85EBCA77u)) >> (32 - SR_HBITS);
}

// Reported positions of one 64-bit word of match bits B, given whether the position before bit 0 was reported:
// in every run of matches the positions at an even distance from the run's start (the run through bit 0 starts one
// earlier when its predecessor was reported).  B + (even run starts) clears exactly the runs that start at even bits.
__device__ __forceinline__ uint64_t sr_alternate(uint64_t B, uint32_t prev)
{
    const uint64_t E = 0x5555555555555555ull;
    uint64_t se = B & ~(B << 1) & E;
    if (prev) se &= ~1ull;
    const uint64_t even_runs = B & ~(B + se);
    return (even_runs & E) | (B & ~even_runs & ~E);
}

// The per-word state map "reported before -> reported at bit 63": the identity for a word of all matches (64 is even),
// a constant otherwise.  Encoded as bit 1 = identity, bit 0 = the constant.
__device__ __forceinline__ uint32_t sr_word_map(uint64_t B) { return B == ~0ull ? 2u : (uint32_t)(sr_alternate(B, 0) >> 63); }
__device__ __forceinline__ uint32_t sr_then(uint32_t a, uint32_t b) { return (b & 2u) ? a : b; }      // a, then b
__device__ __forceinline__ uint32_t sr_apply(uint32_t f, uint32_t r) { return (f & 2u) ? r : (f & 1u); }

// One warp, one pattern, one tile: this lane's two words of reported positions for an incoming flag r, from the warp's
// exclusive scan `pre` of the word maps.
__device__ __forceinline__ void sr_lane_bits(uint64_t b0, uint64_t b1, uint32_t pre, uint32_t r, uint64_t& r0, uint64_t& r1)
{
    r0 = sr_alternate(b0, sr_apply(pre, r));
    r1 = sr_alternate(b1, (uint32_t)(r0 >> 63));
}

template <bool EMIT>
__global__ void __launch_bounds__(SR_THREADS)
k_search_tiles(const uint8_t* __restrict__ chunk, uint64_t chunk_pos, uint64_t valid, uint32_t ntiles,
               const uint8_t* __restrict__ gpat /*[32][256]*/, const uint32_t* __restrict__ ghash /*[2^16 / 32]*/, SrParams P,
               uint32_t* __restrict__ summ /*[npat][ntiles]*/, const uint32_t* __restrict__ toff /*[npat][ntiles]*/,
               SrEmit em, uint32_t* __restrict__ out)
{
    __shared__ __align__(16) uint8_t  s_data[SR_TILE + SR_HALO];
    __shared__ __align__(16) uint8_t  s_pat[JSGPU_SEARCH_MAX_PATTERNS][256];
    __shared__ uint32_t s_hash[(1 << SR_HBITS) / 32];
    __shared__ __align__(16) uint32_t s_match[JSGPU_SEARCH_MAX_PATTERNS][SR_WORDS];
    __shared__ uint32_t s_tin[JSGPU_SEARCH_MAX_PATTERNS];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, npat = P.npat;

    for (uint32_t i = tid; i < (1u << SR_HBITS) / 32; i += SR_THREADS) s_hash[i] = ghash[i];
    for (uint32_t i = tid; i < npat * 256 / 16; i += SR_THREADS) ((uint4*)s_pat)[i] = ((const uint4*)gpat)[i];
    for (uint32_t i = tid; i < JSGPU_SEARCH_MAX_PATTERNS * SR_WORDS; i += SR_THREADS) (&s_match[0][0])[i] = 0;

    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const uint64_t tb = (uint64_t)t * SR_TILE;           // tile start inside the chunk
        __syncthreads();                                      // the previous tile is done with s_data, s_match and s_tin
        if (EMIT) {
            // only tiles that report something inside `cap` are staged again
            int want = 0;
            if (tid < npat) {
                const uint32_t o = toff[(size_t)tid * ntiles + t], s = summ[(size_t)tid * ntiles + t];
                const uint32_t cnt = (o & 1u) ? ((s >> 12) & 0xFFFu) : (s & 0xFFFu);
                want = cnt && (o >> 1) < em.lim[tid];
                s_tin[tid] = o;
            }
            if (!__syncthreads_or(want)) continue;
        }
        for (uint32_t i = tid; i < (SR_TILE + SR_HALO) / 16; i += SR_THREADS) {
            const uint64_t g = tb + 16ull * i;
            uint4 v;
            if (g + 16 <= valid) v = *(const uint4*)(chunk + g);
            else {
                uint8_t b[16];
                for (int j = 0; j < 16; j++) b[j] = (g + j < valid) ? chunk[g + j] : 0;
                memcpy(&v, b, 16);
            }
            ((uint4*)s_data)[i] = v;
        }
        __syncthreads();

        // filter: 16 consecutive positions per thread, windows cut from six registers
        const uint4 a = ((const uint4*)s_data)[tid];
        const uint2 b = *(const uint2*)(s_data + 16 * tid + 16);
        const uint32_t w[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
        int any = 0;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const uint32_t lo = __funnelshift_r(w[i / 4], w[i / 4 + 1], 8 * (i % 4));
            const uint32_t hi = __funnelshift_r(w[i / 4 + 1], w[i / 4 + 2], 8 * (i % 4));
            const uint32_t h = sr_hash(lo, hi);
            if ((s_hash[h >> 5] >> (h & 31)) & 1u) {
                const uint32_t p = 16 * tid + i;
                const int64_t fp = (int64_t)(chunk_pos + tb + p);
                for (uint32_t k = 0; k < npat; k++) {
                    if (P.pre_lo[k] != lo || P.pre_hi[k] != hi || fp < 1 || fp > P.maxp[k]) continue;
                    uint32_t j = 8;
                    const uint32_t L = P.len[k];
                    while (j < L && s_data[p + j] == s_pat[k][j]) j++;
                    if (j == L) { atomicOr(&s_match[k][p >> 5], 1u << (p & 31)); any = 1; }
                }
            }
        }
        if (!__syncthreads_or(any)) {
            if (!EMIT && tid < npat) summ[(size_t)tid * ntiles + t] = 0;
            continue;
        }

        // one warp per pattern: lane l owns positions 128 l .. 128 l + 127 as two 64-bit words
        for (uint32_t k = warp; k < npat; k += SR_THREADS / 32) {
            const uint64_t b0 = ((const uint64_t*)s_match[k])[2 * lane], b1 = ((const uint64_t*)s_match[k])[2 * lane + 1];
            uint32_t f = sr_then(sr_word_map(b0), sr_word_map(b1)), inc = f;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t o = __shfl_up_sync(0xffffffffu, inc, d);
                if (lane >= (uint32_t)d) inc = sr_then(o, inc);
            }
            uint32_t pre = __shfl_up_sync(0xffffffffu, inc, 1);
            if (lane == 0) pre = 2u;
            if (!EMIT) {
                const uint32_t tot = __shfl_sync(0xffffffffu, inc, 31);
                uint64_t r0, r1;
                sr_lane_bits(b0, b1, pre, 0, r0, r1);
                const uint32_t c0 = __reduce_add_sync(0xffffffffu, (uint32_t)(__popcll(r0) + __popcll(r1)));
                sr_lane_bits(b0, b1, pre, 1, r0, r1);
                const uint32_t c1 = __reduce_add_sync(0xffffffffu, (uint32_t)(__popcll(r0) + __popcll(r1)));
                if (lane == 0) summ[(size_t)k * ntiles + t] = c0 | (c1 << 12) | (sr_apply(tot, 0) << 24) | (sr_apply(tot, 1) << 25);
            } else {
                const uint32_t o = s_tin[k];
                uint64_t r0, r1;
                sr_lane_bits(b0, b1, pre, o & 1u, r0, r1);
                const uint32_t n = (uint32_t)(__popcll(r0) + __popcll(r1));
                uint32_t ex = n;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t v = __shfl_up_sync(0xffffffffu, ex, d);
                    if (lane >= (uint32_t)d) ex += v;
                }
                uint32_t j = (o >> 1) + ex - n;                  // chunk-local output index of this lane's first position
                const uint32_t fp0 = (uint32_t)(chunk_pos + tb) + 128 * lane;
                for (int h = 0; h < 2; h++) {
                    uint64_t r = h ? r1 : r0;
                    while (r && j < em.lim[k]) {
                        out[em.base[k] + j] = fp0 + 64 * h + (uint32_t)__ffsll((long long)r) - 1;
                        r &= r - 1; j++;
                    }
                }
            }
            __syncwarp();
            ((uint64_t*)s_match[k])[2 * lane] = 0; ((uint64_t*)s_match[k])[2 * lane + 1] = 0;
        }
    }
}

// One CTA per pattern: chains the tile summaries of a chunk.  A summary is the map "reported before the tile ->
// (count, reported at its last position)" for both inputs; the scan composes them left to right.
struct SrMap { uint32_t o0, o1, c0, c1; };
__device__ __forceinline__ SrMap sr_compose(const SrMap& a, const SrMap& b)    // a, then b
{
    SrMap r;
    r.o0 = a.o0 ? b.o1 : b.o0; r.o1 = a.o1 ? b.o1 : b.o0;
    r.c0 = a.c0 + (a.o0 ? b.c1 : b.c0); r.c1 = a.c1 + (a.o1 ? b.c1 : b.c0);
    return r;
}

__global__ void __launch_bounds__(1024)
k_search_scan(const uint32_t* __restrict__ summ, uint32_t ntiles, uint32_t* __restrict__ toff, uint32_t* __restrict__ chunk_res,
              uint32_t chunk, uint32_t npat)
{
    __shared__ SrMap s_w[32];
    __shared__ uint32_t s_r, s_tot;
    const uint32_t k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // chunk_res[c][k] = {count, outgoing flag}
    if (tid == 0) { s_r = chunk ? chunk_res[2 * ((size_t)(chunk - 1) * npat + k) + 1] : 0u; s_tot = 0; }
    __syncthreads();
    for (uint32_t t0 = 0; t0 < ntiles; t0 += 1024) {
        const uint32_t t = t0 + tid;
        SrMap m = {0u, 1u, 0u, 0u};                            // identity
        if (t < ntiles) {
            const uint32_t s = summ[(size_t)k * ntiles + t];
            m.c0 = s & 0xFFFu; m.c1 = (s >> 12) & 0xFFFu; m.o0 = (s >> 24) & 1u; m.o1 = (s >> 25) & 1u;
        }
        SrMap inc = m;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            SrMap o;
            o.o0 = __shfl_up_sync(0xffffffffu, inc.o0, d); o.o1 = __shfl_up_sync(0xffffffffu, inc.o1, d);
            o.c0 = __shfl_up_sync(0xffffffffu, inc.c0, d); o.c1 = __shfl_up_sync(0xffffffffu, inc.c1, d);
            if (lane >= (uint32_t)d) inc = sr_compose(o, inc);
        }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            SrMap v = s_w[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                SrMap o;
                o.o0 = __shfl_up_sync(0xffffffffu, v.o0, d); o.o1 = __shfl_up_sync(0xffffffffu, v.o1, d);
                o.c0 = __shfl_up_sync(0xffffffffu, v.c0, d); o.c1 = __shfl_up_sync(0xffffffffu, v.c1, d);
                if (lane >= (uint32_t)d) v = sr_compose(o, v);
            }
            s_w[lane] = v;                                    // inclusive over warps
        }
        __syncthreads();
        const uint32_t r = s_r, tot = s_tot;
        SrMap ex = {0u, 1u, 0u, 0u};
        if (warp) ex = s_w[warp - 1];
        SrMap in_warp;                                        // exclusive inside the warp
        in_warp.o0 = __shfl_up_sync(0xffffffffu, inc.o0, 1); in_warp.o1 = __shfl_up_sync(0xffffffffu, inc.o1, 1);
        in_warp.c0 = __shfl_up_sync(0xffffffffu, inc.c0, 1); in_warp.c1 = __shfl_up_sync(0xffffffffu, inc.c1, 1);
        if (lane) ex = sr_compose(ex, in_warp);
        if (t < ntiles) {
            const uint32_t rin = r ? ex.o1 : ex.o0, off = tot + (r ? ex.c1 : ex.c0);
            toff[(size_t)k * ntiles + t] = (off << 1) | rin;
        }
        __syncthreads();
        if (tid == 0) { const SrMap all = s_w[31]; s_tot = tot + (r ? all.c1 : all.c0); s_r = r ? all.o1 : all.o0; }
        __syncthreads();
    }
    if (tid == 0) { chunk_res[2 * ((size_t)chunk * npat + k)] = s_tot; chunk_res[2 * ((size_t)chunk * npat + k) + 1] = s_r; }
}

// ---- host side -------------------------------------------------------------------------------------------------------
struct JsSearch {
    int device = -1;
    cudaStream_t st[2] = {nullptr, nullptr};
    cudaEvent_t copied[2] = {nullptr, nullptr}, scanned[2] = {nullptr, nullptr};
    uint8_t* pin[2] = {nullptr, nullptr}; size_t pin_cap = 0;
    uint8_t* dbuf[2] = {nullptr, nullptr}; size_t dbuf_cap = 0;
    uint32_t* dsum[2] = {nullptr, nullptr}; uint32_t* doff[2] = {nullptr, nullptr}; size_t tile_cap = 0;
    uint8_t* dpat = nullptr; uint32_t* dhash = nullptr;
    uint32_t* dres = nullptr; size_t res_cap = 0;
    uint32_t* dout = nullptr; size_t out_cap = 0;
    uint32_t* dfind = nullptr; uint32_t* hfind = nullptr;   // jsgpu_find_value: one result word per slot, device and pinned host
    uint32_t* dfa[2] = {nullptr, nullptr}; size_t fa_cap = 0;   // jsgpu_find_all: per-CTA counts and output indices per slot
};

void js_search_free(JsSearch* s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    for (int i = 0; i < 2; i++) {
        if (s->st[i]) cudaStreamSynchronize(s->st[i]);
        cudaFreeHost(s->pin[i]); cudaFree(s->dbuf[i]); cudaFree(s->dsum[i]); cudaFree(s->doff[i]); cudaFree(s->dfa[i]);
        if (s->copied[i]) cudaEventDestroy(s->copied[i]);
        if (s->scanned[i]) cudaEventDestroy(s->scanned[i]);
        if (s->st[i]) cudaStreamDestroy(s->st[i]);
    }
    cudaFree(s->dpat); cudaFree(s->dhash); cudaFree(s->dres); cudaFree(s->dout); cudaFree(s->dfind); cudaFreeHost(s->hfind);
    delete s;
}

static uint64_t sr_chunk_bytes()
{
    uint64_t c = 64ull << 20;
    if (const char* e = getenv("JSGPU_SEARCH_CHUNK_BYTES")) { const unsigned long long v = strtoull(e, nullptr, 10); if (v) c = v; }
    c = (c + SR_TILE - 1) / SR_TILE * SR_TILE;
    return std::min<uint64_t>(c, 128ull << 20);               // keeps every per-chunk count and output index within 32 bits
}

#define SR_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { err = std::string(#call " failed: ") + cudaGetErrorString(e_); \
                         return e_ == cudaErrorMemoryAllocation ? JSGPU_ENOMEM : JSGPU_ECUDA; } } while (0)

template <typename T> static cudaError_t sr_grow(T*& p, size_t& cap, size_t n)
{
    if (n <= cap) return cudaSuccess;
    cudaFree(p); p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc((void**)&p, n * sizeof(T));
    if (e == cudaSuccess) cap = n;
    return e;
}

#define SR_TRY(call) do { const int r_ = (call); if (r_ != JSGPU_OK) return r_; } while (0)

// the search's streams, events and small buffers, created on the context's first search
static int sr_open(JsSearch** ps, int device, std::string& err)
{
    cudaSetDevice(device);
    if (*ps) return JSGPU_OK;
    JsSearch* s = new JsSearch(); s->device = device;
    *ps = s;
    for (int i = 0; i < 2; i++) {
        SR_CK(cudaStreamCreateWithFlags(&s->st[i], cudaStreamNonBlocking));
        SR_CK(cudaEventCreateWithFlags(&s->copied[i], cudaEventDisableTiming));
        SR_CK(cudaEventCreateWithFlags(&s->scanned[i], cudaEventDisableTiming));
    }
    size_t c0 = 0, c1 = 0, c2 = 0;
    SR_CK(sr_grow(s->dpat, c0, (size_t)JSGPU_SEARCH_MAX_PATTERNS * 256));
    SR_CK(sr_grow(s->dhash, c1, (size_t)(1u << SR_HBITS) / 32));
    SR_CK(sr_grow(s->dfind, c2, 2));
    SR_CK(cudaMallocHost((void**)&s->hfind, 2 * sizeof(uint32_t)));
    return JSGPU_OK;
}

// two pinned staging buffers of at least `pin` bytes and two device chunk buffers of at least `dev` bytes
static int sr_reserve(JsSearch* s, size_t pin, size_t dev, std::string& err)
{
    if (s->pin_cap < pin) {
        for (int i = 0; i < 2; i++) { cudaFreeHost(s->pin[i]); s->pin[i] = nullptr; }
        s->pin_cap = 0;
        for (int i = 0; i < 2; i++) SR_CK(cudaMallocHost((void**)&s->pin[i], pin));
        s->pin_cap = pin;
    }
    if (s->dbuf_cap < dev) {
        for (int i = 0; i < 2; i++) { cudaFree(s->dbuf[i]); s->dbuf[i] = nullptr; }
        s->dbuf_cap = 0;
        for (int i = 0; i < 2; i++) SR_CK(cudaMalloc((void**)&s->dbuf[i], dev));
        s->dbuf_cap = dev;
    }
    return JSGPU_OK;
}

int js_search_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, const uint8_t* pats, const uint32_t* lens,
                  uint32_t npat, uint64_t* counts, uint32_t* pos, uint64_t cap, std::string& err)
{
    for (uint32_t k = 0; k < npat; k++) counts[k] = 0;
    if (n == 0) return JSGPU_OK;
    SR_TRY(sr_open(ps, device, err));
    JsSearch* s = *ps;

    // patterns, their prefix hash and the reporting limits
    SrParams P; memset(&P, 0, sizeof P);
    P.npat = npat;
    std::vector<uint8_t> hpat((size_t)JSGPU_SEARCH_MAX_PATTERNS * 256, 0);
    std::vector<uint32_t> hhash((1u << SR_HBITS) / 32, 0);
    for (uint32_t k = 0, o = 0; k < npat; o += lens[k], k++) {
        memcpy(&hpat[(size_t)k * 256], pats + o, lens[k]);
        P.len[k] = lens[k]; P.maxlen = std::max(P.maxlen, lens[k]);
        P.maxp[k] = (int64_t)n - 2 * (int64_t)lens[k] + 2;
        memcpy(&P.pre_lo[k], pats + o, 4); memcpy(&P.pre_hi[k], pats + o + 4, 4);
        const uint32_t h = ((P.pre_lo[k] * 0x9E3779B1u) ^ (P.pre_hi[k] * 0x85EBCA77u)) >> (32 - SR_HBITS);
        hhash[h >> 5] |= 1u << (h & 31);
    }
    SR_CK(cudaMemcpyAsync(s->dpat, hpat.data(), hpat.size(), cudaMemcpyHostToDevice, s->st[0]));
    SR_CK(cudaMemcpyAsync(s->dhash, hhash.data(), hhash.size() * 4, cudaMemcpyHostToDevice, s->st[0]));
    SR_CK(cudaStreamSynchronize(s->st[0]));

    const uint64_t chunk = std::min<uint64_t>(sr_chunk_bytes(), (n + SR_TILE - 1) / SR_TILE * SR_TILE);
    const uint32_t nchunks = (uint32_t)((n + chunk - 1) / chunk);
    const uint32_t tiles = (uint32_t)(chunk / SR_TILE);
    const size_t span = chunk + P.maxlen - 1;                 // bytes uploaded per chunk
    SR_TRY(sr_reserve(s, span, span, err));
    const size_t tneed = (size_t)tiles * npat;
    if (s->tile_cap < tneed) {
        for (int i = 0; i < 2; i++) { cudaFree(s->dsum[i]); cudaFree(s->doff[i]); s->dsum[i] = s->doff[i] = nullptr; }
        s->tile_cap = 0;
        for (int i = 0; i < 2; i++) { SR_CK(cudaMalloc((void**)&s->dsum[i], tneed * 4)); SR_CK(cudaMalloc((void**)&s->doff[i], tneed * 4)); }
        s->tile_cap = tneed;
    }
    SR_CK(sr_grow(s->dres, s->res_cap, (size_t)nchunks * npat * 2));

    int occ = 0;
    SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_search_tiles<false>, SR_THREADS, 0));
    const uint32_t grid = std::max(1u, std::min<uint32_t>(tiles, (uint32_t)(std::max(occ, 1) * sm_count)));
    SrEmit none; memset(&none, 0, sizeof none);

    // stage chunk c into slot c & 1 and search it; `scan_after` orders the summary chain across the two streams
    int resident = -1;
    auto run_chunk = [&](uint32_t c, bool emit, const SrEmit& em, int prev_slot_scan) -> int {
        const int sl = c & 1;
        const uint64_t c0 = (uint64_t)c * chunk, valid = std::min<uint64_t>(span, n - c0);
        if (resident != (int)c) {
            SR_CK(cudaEventSynchronize(s->copied[sl]));       // the pinned buffer's previous upload has left
            memcpy(s->pin[sl], data + c0, valid);
            SR_CK(cudaMemcpyAsync(s->dbuf[sl], s->pin[sl], valid, cudaMemcpyHostToDevice, s->st[sl]));
            SR_CK(cudaEventRecord(s->copied[sl], s->st[sl]));
            resident = (int)c;
        }
        const uint32_t nt = (uint32_t)std::min<uint64_t>(tiles, (n - c0 + SR_TILE - 1) / SR_TILE);
        k_search_tiles<false><<<std::min(grid, nt), SR_THREADS, 0, s->st[sl]>>>(s->dbuf[sl], c0, valid, nt, s->dpat, s->dhash, P,
                                                                                s->dsum[sl], nullptr, none, nullptr);
        if (prev_slot_scan >= 0) SR_CK(cudaStreamWaitEvent(s->st[sl], s->scanned[prev_slot_scan], 0));
        k_search_scan<<<npat, 1024, 0, s->st[sl]>>>(s->dsum[sl], nt, s->doff[sl], s->dres, c, npat);
        SR_CK(cudaEventRecord(s->scanned[sl], s->st[sl]));
        if (emit)
            k_search_tiles<true><<<std::min(grid, nt), SR_THREADS, 0, s->st[sl]>>>(s->dbuf[sl], c0, valid, nt, s->dpat, s->dhash, P,
                                                                                   s->dsum[sl], s->doff[sl], em, s->dout);
        SR_CK(cudaGetLastError());
        return JSGPU_OK;
    };

    // pass 1: counts per chunk and pattern
    for (uint32_t c = 0; c < nchunks; c++) {
        int r = run_chunk(c, false, none, c ? (int)((c - 1) & 1) : -1);
        if (r) return r;
    }
    std::vector<uint32_t> res((size_t)nchunks * npat * 2);
    SR_CK(cudaStreamSynchronize(s->st[0])); SR_CK(cudaStreamSynchronize(s->st[1]));
    SR_CK(cudaMemcpy(res.data(), s->dres, res.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t c = 0; c < nchunks; c++) for (uint32_t k = 0; k < npat; k++) counts[k] += res[2 * ((size_t)c * npat + k)];

    // pass 2: chunks with positions inside `cap`, written in place (pattern k's list follows pattern k-1's)
    if (cap && pos) {
        std::vector<uint64_t> first(npat), run(npat, 0);      // global index of pattern k's first position; its positions before chunk c
        uint64_t acc = 0;
        for (uint32_t k = 0; k < npat; k++) { first[k] = acc; acc += counts[k]; }
        for (uint32_t c = 0; c < nchunks; c++) {
            SrEmit em; memset(&em, 0, sizeof em);
            uint64_t total = 0;
            for (uint32_t k = 0; k < npat; k++) {
                const uint64_t cnt = res[2 * ((size_t)c * npat + k)], g = first[k] + run[k];
                const uint64_t keep = g >= cap ? 0 : std::min<uint64_t>(cnt, cap - g);
                em.lim[k] = (uint32_t)keep; em.base[k] = (uint32_t)total; total += keep;
            }
            if (total) {
                SR_CK(sr_grow(s->dout, s->out_cap, (size_t)total));
                int r = run_chunk(c, true, em, c ? (int)((c - 1) & 1) : -1);
                if (r) return r;
                SR_CK(cudaStreamSynchronize(s->st[c & 1]));
                std::vector<uint32_t> h(total);
                SR_CK(cudaMemcpy(h.data(), s->dout, total * 4, cudaMemcpyDeviceToHost));
                for (uint32_t k = 0; k < npat; k++)
                    if (em.lim[k]) memcpy(pos + first[k] + run[k], h.data() + em.base[k], (size_t)em.lim[k] * 4);
            }
            for (uint32_t k = 0; k < npat; k++) run[k] += res[2 * ((size_t)c * npat + k)];
        }
    }
    SR_CK(cudaStreamSynchronize(s->st[0])); SR_CK(cudaStreamSynchronize(s->st[1]));
    return JSGPU_OK;
}

// ---- value search (jsgpu_find_value, include/jsgpu.h) -----------------------------------------------------------------
// CwindowBuf::BufSearch (WindowBuf.cpp:149-212) compares the big-endian value of the `len` bytes at each position with the
// value, one position at a time, forward from start + 1 or backward from start - 1, and stops at the first match.  Here the
// positions whose bytes all lie inside the file are searched on the device, chunk by chunk in search order; the few that
// read past the end of the file (as 0, WindowBuf.cpp:704-711) are tested on the host.
#define FV_THREADS 256
#define FV_TILE    (FV_THREADS * 16)     // 16 consecutive positions per thread

// Positions 0 .. npos-1 of one chunk: buf holds their npos + len - 1 bytes and is readable up to 20 bytes past the last
// 16-byte group.  A position matches when its four bytes, little-endian and masked to len bytes, equal `pat`.
// The match mask of positions p0 .. p0 + 15 (p0 a multiple of 16): five 32-bit loads, the windows cut by funnel shifts.
__device__ __forceinline__ uint32_t fv_match16(const uint8_t* __restrict__ buf, uint32_t p0, uint32_t npos, uint32_t pat, uint32_t mask)
{
    uint32_t m = 0;
    if (p0 < npos) {
        const uint4 a = *(const uint4*)(buf + p0);
        const uint32_t w[5] = {a.x, a.y, a.z, a.w, *(const uint32_t*)(buf + p0 + 16)};
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const uint32_t v = (k % 4) ? __funnelshift_r(w[k / 4], w[k / 4 + 1], 8 * (k % 4)) : w[k / 4];
            if ((v & mask) == pat) m |= 1u << k;
        }
        if (npos - p0 < 16) m &= (1u << (npos - p0)) - 1u;
    }
    return m;
}

// res receives the lowest match (forward) or the highest match + 1 (reverse) if it beats what is there.
__global__ void __launch_bounds__(FV_THREADS)
k_find_value(const uint8_t* __restrict__ buf, uint32_t npos, uint32_t pat, uint32_t mask, int forward, uint32_t* __restrict__ res)
{
    __shared__ uint32_t s_best;                              // forward: lowest match, ~0 for none; reverse: highest + 1, 0 for none
    const uint32_t tid = threadIdx.x, lane = tid & 31, none = forward ? 0xFFFFFFFFu : 0u;
    if (tid == 0) s_best = none;
    __syncthreads();
    const uint32_t ntiles = (npos + FV_TILE - 1) / FV_TILE;
    // tiles in search order, so that a CTA can stop at its first tile with a match
    for (uint32_t i = blockIdx.x; i < ntiles; i += gridDim.x) {
        const uint32_t t = forward ? i : ntiles - 1 - i;
        const uint32_t p0 = t * FV_TILE + 16 * tid;
        const uint32_t m = fv_match16(buf, p0, npos, pat, mask);
        const uint32_t vote = __ballot_sync(0xffffffffu, m != 0);
        if (vote && lane == (uint32_t)(forward ? __ffs(vote) - 1 : 31 - __clz(vote))) {
            if (forward) atomicMin(&s_best, p0 + __ffs(m) - 1);
            else         atomicMax(&s_best, p0 + (31 - __clz(m)) + 1);
        }
        if (__syncthreads_or(m != 0)) break;                 // every later tile of this CTA lies further in search order
    }
    __syncthreads();
    if (tid == 0 && s_best != none) {
        if (forward) atomicMin(res, s_best);
        else         atomicMax(res, s_best);
    }
}

int js_find_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, uint64_t start, uint32_t value,
                uint32_t len, int forward, const jsgpu_overlay* ovl, uint32_t novl, int* found, uint64_t* found_pos, std::string& err)
{
    // Buf(): the file byte, 0 past EOF, replaced by the last enabled overlay that covers it (WindowBuf.cpp:655-681)
    auto byte_at = [&](uint64_t q) {
        uint8_t b = q < n ? data[q] : 0;
        for (uint32_t k = 0; k < novl; k++) if (q >= ovl[k].start && q - ovl[k].start < ovl[k].len) b = ovl[k].data[q - ovl[k].start];
        return b;
    };
    auto test = [&](uint64_t p) { uint32_t v = 0; for (uint32_t i = 0; i < len; i++) v = (v << 8) | byte_at(p + i); return v == value; };
    const uint32_t mask = len == 4 ? 0xFFFFFFFFu : (1u << (8 * len)) - 1u;
    const bool possible = (value & ~mask) == 0;               // a value wider than len bytes never matches
    const int64_t inside = (int64_t)n - (int64_t)len;         // the last position whose bytes all lie in the file
    *found = 0;

    // the positions the device searches, [lo, hi], and what the host tests around them
    int64_t lo = 0, hi = -1;
    if (forward) {
        // start + 1, start + 2, ... up to and including the first position that reads past EOF (or start + 1 alone)
        const int64_t first = (int64_t)start + 1, last = std::max(first, inside + 1);
        *found_pos = (uint64_t)last;
        if (!possible) return JSGPU_OK;
        lo = first; hi = last - 1;
    } else {
        *found_pos = 0;                                       // the reference stops at 0 (from 0 it tests 0 once)
        if (!possible) return JSGPU_OK;
        int64_t p = start ? (int64_t)start - 1 : 0;
        // positions that read past EOF, from the top: past the file and every overlay the bytes are all 0
        while (p > inside && p >= 0) {
            bool touched = p < (int64_t)n;
            int64_t next = (int64_t)n - 1;                    // the next lower position whose bytes can differ from 0
            for (uint32_t k = 0; k < novl; k++) {
                const int64_t s0 = (int64_t)ovl[k].start - (int64_t)len + 1, s1 = (int64_t)(ovl[k].start + ovl[k].len) - 1;
                if (p >= s0 && p <= s1) touched = true;
                if (s0 <= p - 1) next = std::max(next, std::min(s1, p - 1));
            }
            if (touched ? test((uint64_t)p) : value == 0) { *found = 1; *found_pos = (uint64_t)p; return JSGPU_OK; }
            if (!start) return JSGPU_OK;
            p = touched ? p - 1 : next;
        }
        if (!start) { *found = test(0); return JSGPU_OK; }
        lo = 0; hi = p;
    }

    if (hi >= lo) {
        SR_TRY(sr_open(ps, device, err));
        JsSearch* s = *ps;
        const uint64_t range = (uint64_t)(hi - lo + 1);
        const uint64_t chunk = std::min<uint64_t>(sr_chunk_bytes(), (range + FV_TILE - 1) / FV_TILE * FV_TILE);
        const uint64_t nchunks = (range + chunk - 1) / chunk;
        SR_TRY(sr_reserve(s, chunk + 3, chunk + 64, err));
        int occ = 0;
        SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_find_value, FV_THREADS, 0));
        const uint32_t grid_max = (uint32_t)(std::max(occ, 1) * sm_count);
        const uint32_t pat = __builtin_bswap32(value) >> (32 - 8 * len);      // the bytes in file order, little-endian
        // chunk c in search order: positions [plo, phi], bytes [plo, phi + len - 1] (its len - 1 halo bytes lie in the file)
        auto bounds = [&](uint64_t c, uint64_t& plo, uint64_t& phi) {
            if (forward) { plo = (uint64_t)lo + c * chunk; phi = std::min<uint64_t>((uint64_t)hi, plo + chunk - 1); }
            else         { phi = (uint64_t)hi - c * chunk; plo = phi + 1 > (uint64_t)lo + chunk ? phi + 1 - chunk : (uint64_t)lo; }
        };
        auto stage = [&](uint64_t c) {
            uint64_t plo, phi; bounds(c, plo, phi);
            const uint64_t nb = phi - plo + len;
            uint8_t* dst = s->pin[c & 1];
            memcpy(dst, data + plo, nb);
            for (uint32_t k = 0; k < novl; k++) {                  // installed order: the last overlay wins
                const uint64_t a = std::max<uint64_t>(ovl[k].start, plo), b = std::min<uint64_t>(ovl[k].start + ovl[k].len, plo + nb);
                if (a < b) memcpy(dst + (a - plo), ovl[k].data + (a - ovl[k].start), b - a);
            }
        };
        // The host stages chunk c + 1 while the device searches chunk c; chunk c + 1 goes to the device only if c has no match.
        stage(0);
        for (uint64_t c = 0; c < nchunks; c++) {
            const int sl = (int)(c & 1);
            uint64_t plo, phi; bounds(c, plo, phi);
            const uint32_t npos = (uint32_t)(phi - plo + 1);
            SR_CK(cudaMemcpyAsync(s->dbuf[sl], s->pin[sl], npos + len - 1, cudaMemcpyHostToDevice, s->st[sl]));
            SR_CK(cudaMemsetAsync(s->dfind + sl, forward ? 0xFF : 0, 4, s->st[sl]));
            const uint32_t grid = std::max(1u, std::min(grid_max, (npos + FV_TILE - 1) / FV_TILE));
            k_find_value<<<grid, FV_THREADS, 0, s->st[sl]>>>(s->dbuf[sl], npos, pat, mask, forward, s->dfind + sl);
            SR_CK(cudaGetLastError());
            SR_CK(cudaMemcpyAsync(s->hfind + sl, s->dfind + sl, 4, cudaMemcpyDeviceToHost, s->st[sl]));
            SR_CK(cudaEventRecord(s->copied[sl], s->st[sl]));
            if (c + 1 < nchunks) stage(c + 1);                    // the other slot's chunk finished in the previous round
            SR_CK(cudaEventSynchronize(s->copied[sl]));
            const uint32_t r = s->hfind[sl];
            if (forward ? r != 0xFFFFFFFFu : r != 0u) {
                *found = 1; *found_pos = plo + (forward ? r : r - 1);
                return JSGPU_OK;
            }
        }
    }
    if (forward) *found = test(*found_pos);                  // the last position, which reads past EOF
    return JSGPU_OK;
}

// ---- every match of a value (jsgpu_find_all, include/jsgpu.h) ----------------------------------------------------------
// Each chunk is uploaded once and stays resident while three kernels run on it: k_find_all<false> counts the matches of
// each CTA's run of consecutive tiles, k_find_all_scan turns the counts into output indices from the running total kept on
// the device, and k_find_all<true> writes the positions in file order.  CTA b owns tiles [b * per, (b + 1) * per).
template <bool EMIT>
__global__ void __launch_bounds__(FV_THREADS)
k_find_all(const uint8_t* __restrict__ buf, uint32_t npos, uint32_t pat, uint32_t mask, uint32_t per, uint32_t chunk_pos,
           uint32_t* __restrict__ cta /*[2][gridDim.x]: counts, then first output index*/, uint32_t* __restrict__ out, uint64_t cap)
{
    __shared__ uint32_t s_w[FV_THREADS / 32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t ntiles = (npos + FV_TILE - 1) / FV_TILE;
    const uint32_t t0 = blockIdx.x * per, t1 = min(ntiles, t0 + per);
    if (!EMIT) {
        uint32_t c = 0;
        for (uint32_t t = t0; t < t1; t++) c += __popc(fv_match16(buf, t * FV_TILE + 16 * tid, npos, pat, mask));
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) s_w[warp] = c;
        __syncthreads();
        if (tid == 0) {
            uint32_t sum = 0;
            for (int k = 0; k < FV_THREADS / 32; k++) sum += s_w[k];
            cta[blockIdx.x] = sum;
        }
        return;
    }
    uint32_t j = cta[gridDim.x + blockIdx.x];                // this CTA's first output index
    if (cta[blockIdx.x] == 0 || j >= cap) return;
    for (uint32_t t = t0; t < t1 && j < cap; t++) {
        uint32_t m = fv_match16(buf, t * FV_TILE + 16 * tid, npos, pat, mask);
        const uint32_t c = __popc(m);
        uint32_t inc = c;                                     // inclusive scan over the warp, then over the warps
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += v;
        }
        __syncthreads();                                      // the previous tile is done with s_w
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        uint32_t before = 0, tot = 0;
#pragma unroll
        for (int k = 0; k < FV_THREADS / 32; k++) { const uint32_t v = s_w[k]; before += (uint32_t)k < warp ? v : 0u; tot += v; }
        uint64_t o = (uint64_t)j + before + inc - c;
        const uint32_t p = chunk_pos + t * FV_TILE + 16 * tid;
        while (m && o < cap) { out[o++] = p + (uint32_t)__ffs((int)m) - 1; m &= m - 1; }
        j += tot;
    }
}

// One CTA: the first output index of every CTA of the chunk, from the running total, which it then advances.
__global__ void __launch_bounds__(1024)
k_find_all_scan(uint32_t* __restrict__ cta, uint32_t ncta, uint32_t* __restrict__ total)
{
    __shared__ uint32_t s_w[32], s_run;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_run = *total;
    for (uint32_t b0 = 0; b0 < ncta; b0 += 1024) {
        __syncthreads();
        const uint32_t b = b0 + tid, c = b < ncta ? cta[b] : 0u;
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= (uint32_t)d) inc += v;
        }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        uint32_t before = 0, tot = 0;
        for (uint32_t k = 0; k < 32; k++) { const uint32_t v = s_w[k]; before += k < warp ? v : 0u; tot += v; }
        if (b < ncta) cta[ncta + b] = s_run + before + inc - c;
        __syncthreads();
        if (tid == 0) s_run += tot;
    }
    __syncthreads();
    if (tid == 0) *total = s_run;
}

int js_find_all_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, uint32_t value, uint32_t len,
                    uint64_t* count, uint32_t* pos, uint64_t cap, std::string& err)
{
    *count = 0;
    const uint32_t mask = len == 4 ? 0xFFFFFFFFu : (1u << (8 * len)) - 1u;
    if (n < len || (value & ~mask)) return JSGPU_OK;         // no position, or a value wider than len bytes
    SR_TRY(sr_open(ps, device, err));
    JsSearch* s = *ps;
    const uint64_t npos_all = n - len + 1;
    const uint64_t chunk = std::min<uint64_t>(sr_chunk_bytes(), (npos_all + FV_TILE - 1) / FV_TILE * FV_TILE);
    const uint64_t nchunks = (npos_all + chunk - 1) / chunk;
    SR_TRY(sr_reserve(s, chunk + 3, chunk + 64, err));
    int occ = 0;
    SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_find_all<true>, FV_THREADS, 0));
    const uint32_t grid_max = (uint32_t)(std::max(occ, 1) * sm_count);
    if (s->fa_cap < 2 * (size_t)grid_max) {
        for (int i = 0; i < 2; i++) { cudaFree(s->dfa[i]); s->dfa[i] = nullptr; }
        s->fa_cap = 0;
        for (int i = 0; i < 2; i++) SR_CK(cudaMalloc((void**)&s->dfa[i], 2 * (size_t)grid_max * 4));
        s->fa_cap = 2 * (size_t)grid_max;
    }
    const uint64_t keep = std::min<uint64_t>(cap, npos_all);  // positions the device list can hold
    if (keep) SR_CK(sr_grow(s->dout, s->out_cap, (size_t)keep));
    const uint32_t pat = __builtin_bswap32(value) >> (32 - 8 * len);      // the bytes in file order, little-endian
    uint32_t* const total = s->dfind;                                     // the running count (the value search's result word)
    SR_CK(cudaMemsetAsync(total, 0, 4, s->st[0]));
    SR_CK(cudaEventRecord(s->scanned[1], s->st[0]));                      // chunk 0's scan follows the reset

    for (uint64_t c = 0; c < nchunks; c++) {
        const int sl = (int)(c & 1);
        const uint64_t plo = c * chunk;
        const uint32_t npos = (uint32_t)std::min<uint64_t>(chunk, npos_all - plo);
        SR_CK(cudaEventSynchronize(s->copied[sl]));           // the pinned buffer's previous upload has left
        memcpy(s->pin[sl], data + plo, npos + len - 1);
        SR_CK(cudaMemcpyAsync(s->dbuf[sl], s->pin[sl], npos + len - 1, cudaMemcpyHostToDevice, s->st[sl]));
        SR_CK(cudaEventRecord(s->copied[sl], s->st[sl]));
        const uint32_t ntiles = (npos + FV_TILE - 1) / FV_TILE;
        const uint32_t grid = std::max(1u, std::min(grid_max, ntiles)), per = (ntiles + grid - 1) / grid;
        k_find_all<false><<<grid, FV_THREADS, 0, s->st[sl]>>>(s->dbuf[sl], npos, pat, mask, per, (uint32_t)plo, s->dfa[sl], nullptr, 0);
        SR_CK(cudaStreamWaitEvent(s->st[sl], s->scanned[sl ^ 1], 0));  // the previous chunk has advanced the total
        k_find_all_scan<<<1, 1024, 0, s->st[sl]>>>(s->dfa[sl], grid, total);
        SR_CK(cudaEventRecord(s->scanned[sl], s->st[sl]));
        if (keep)
            k_find_all<true><<<grid, FV_THREADS, 0, s->st[sl]>>>(s->dbuf[sl], npos, pat, mask, per, (uint32_t)plo, s->dfa[sl], s->dout, keep);
        SR_CK(cudaGetLastError());
    }
    SR_CK(cudaStreamSynchronize(s->st[0])); SR_CK(cudaStreamSynchronize(s->st[1]));
    uint32_t tot = 0;
    SR_CK(cudaMemcpy(&tot, total, 4, cudaMemcpyDeviceToHost));
    *count = tot;
    const uint64_t got = std::min<uint64_t>(tot, keep);
    if (got) SR_CK(cudaMemcpy(pos, s->dout, got * 4, cudaMemcpyDeviceToHost));
    return JSGPU_OK;
}
