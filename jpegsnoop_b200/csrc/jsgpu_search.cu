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
// The first-match value search of Img Search Fwd / Rev (jsgpu_find_value), the every-match value search (jsgpu_find_all)
// and the extract walk's marker search (jsgpu_find_markers), all at the end of the file, share them.
#include "jsgpu_internal.h"
#include "jsgpu_scan.cuh"
#include <cstdlib>
#include <cstring>
#include <vector>
#include <algorithm>
#include <memory>

#define SR_THREADS  256                  // threads per CTA of the tile kernels
#define SR_TILE     (SR_THREADS * 16)    // positions per tile: 16 consecutive positions per thread
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
            uint32_t inc;
            const uint32_t pre = js_warp_scan(sr_then(sr_word_map(b0), sr_word_map(b1)), 2u, sr_then, inc);
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
                uint32_t n_inc;                                  // j: chunk-local output index of this lane's first position
                uint32_t j = (o >> 1) + js_warp_scan((uint32_t)(__popcll(r0) + __popcll(r1)), 0u, js_add, n_inc);
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
    __shared__ SrMap s_w[33];
    const uint32_t k = blockIdx.x, tid = threadIdx.x;
    const SrMap id = {0u, 1u, 0u, 0u};
    // chunk_res[c][k] = {count, outgoing flag}; r: the flag the chunk starts with
    const uint32_t r = chunk ? chunk_res[2 * ((size_t)(chunk - 1) * npat + k) + 1] : 0u;
    SrMap all = id;                                           // the map of the tiles scanned so far
    for (uint32_t t0 = 0; t0 < ntiles; t0 += 1024) {
        const uint32_t t = t0 + tid;
        SrMap m = id;
        if (t < ntiles) {
            const uint32_t s = summ[(size_t)k * ntiles + t];
            m.c0 = s & 0xFFFu; m.c1 = (s >> 12) & 0xFFFu; m.o0 = (s >> 24) & 1u; m.o1 = (s >> 25) & 1u;
        }
        const SrMap ex = js_block_scan<1024>(m, id, sr_compose, all, s_w);
        if (t < ntiles) toff[(size_t)k * ntiles + t] = ((r ? ex.c1 : ex.c0) << 1) | (r ? ex.o1 : ex.o0);
    }
    if (tid == 0) {
        chunk_res[2 * ((size_t)chunk * npat + k)] = r ? all.c1 : all.c0;
        chunk_res[2 * ((size_t)chunk * npat + k) + 1] = r ? all.o1 : all.o0;
    }
}

// ---- host side: one chunk pipeline for the three searches --------------------------------------------------------------
// Two slots, each a pinned staging buffer, a device chunk buffer and a stream: the host stages chunk k + 1 into one slot
// while the device searches chunk k from the other.  copied[i] follows slot i's last upload; scanned[i] its last scan
// kernel, through which the scans of consecutive chunks are chained across the two streams.
struct JsSearch {
    int device = -1;
    cudaStream_t st[2] = {};
    cudaEvent_t copied[2] = {}, scanned[2] = {};
    PinBuf pin[2];
    DevBuf buf[2];
    DevBuf sum[2], off[2];                  // jsgpu_search_bytes: tile summaries and output offsets per slot ...
    DevBuf pat, hash, res;                  // ... the patterns, their prefix hash, and each chunk's counts and outgoing flags
    DevBuf out;                             // jsgpu_search_bytes (one chunk's) and jsgpu_find_all: the positions
    DevBuf find; PinBuf hfind;              // jsgpu_find_value: one result word per slot, device and pinned host
    DevBuf cta[2], total;                   // jsgpu_find_all: per slot the per-CTA counts and output indices; the running count
    ~JsSearch()
    {
        for (int i = 0; i < 2; i++) {
            if (copied[i]) cudaEventDestroy(copied[i]);
            if (scanned[i]) cudaEventDestroy(scanned[i]);
            if (st[i]) cudaStreamDestroy(st[i]);
        }
    }
};

void js_search_free(JsSearch* s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    for (cudaStream_t t : s->st) cudaStreamSynchronize(t);
    delete s;
}

static uint64_t sr_chunk_bytes()
{
    uint64_t c = 64ull << 20;
    if (const char* e = getenv("JSGPU_SEARCH_CHUNK_BYTES")) { const unsigned long long v = strtoull(e, nullptr, 10); if (v) c = v; }
    c = (c + SR_TILE - 1) / SR_TILE * SR_TILE;
    return std::min<uint64_t>(c, 128ull << 20);               // keeps every per-chunk count and output index within 32 bits
}

// The positions lo .. lo + npos - 1 in chunks of `size` (a multiple of the tile), in search order: upward, or from the top
// when `down`.  Chunk c's bytes are those of its positions and the `halo` bytes after them, as far as the file's n go.
struct SrChunks {
    uint64_t n, lo, npos, size, count;
    uint32_t halo;
    bool down;
    SrChunks(uint64_t n_, uint64_t lo_, uint64_t npos_, uint32_t halo_, bool down_)
        : n(n_), lo(lo_), npos(npos_), size(std::min<uint64_t>(sr_chunk_bytes(), (npos_ + SR_TILE - 1) / SR_TILE * SR_TILE)),
          count((npos_ + size - 1) / size), halo(halo_), down(down_) {}
    uint32_t positions(uint64_t c) const { return (uint32_t)std::min(size, npos - c * size); }
    uint64_t first(uint64_t c) const { return lo + (down ? npos - c * size - positions(c) : c * size); }
    uint64_t bytes(uint64_t c) const { return std::min<uint64_t>(positions(c) + halo, n - first(c)); }
};

#define SR_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { err = std::string(#call " failed: ") + cudaGetErrorString(e_); \
                         return e_ == cudaErrorMemoryAllocation ? JSGPU_ENOMEM : JSGPU_ECUDA; } } while (0)
#define SR_TRY(call) do { const int r_ = (call); if (r_ != JSGPU_OK) return r_; } while (0)

// The context's search, made on its first use, with both slots able to take any chunk of `ch`.  The device chunk buffers
// stay readable 64 bytes past a chunk's bytes: fv_match16 reads up to 19.
static int sr_open(JsSearch** ps, int device, const SrChunks& ch, std::string& err)
{
    cudaSetDevice(device);
    if (!*ps) {
        std::unique_ptr<JsSearch> s(new JsSearch());
        s->device = device;
        for (int i = 0; i < 2; i++) {
            SR_CK(cudaStreamCreateWithFlags(&s->st[i], cudaStreamNonBlocking));
            SR_CK(cudaEventCreateWithFlags(&s->copied[i], cudaEventDisableTiming));
            SR_CK(cudaEventCreateWithFlags(&s->scanned[i], cudaEventDisableTiming));
        }
        *ps = s.release();
    }
    for (int i = 0; i < 2; i++) {
        SR_CK((*ps)->pin[i].reserve(ch.size + ch.halo));
        SR_CK((*ps)->buf[i].reserve(ch.size + ch.halo + 64));
    }
    return JSGPU_OK;
}

// Chunk c's bytes, with the overlays patched in (in installed order: the last one wins), into its slot's pinned buffer,
// once that buffer's previous upload has left.
static int sr_stage(JsSearch* s, const SrChunks& ch, uint64_t c, const uint8_t* data, const jsgpu_overlay* ovl, uint32_t novl,
                    std::string& err)
{
    const uint64_t plo = ch.first(c), nb = ch.bytes(c);
    uint8_t* dst = s->pin[c & 1].as<uint8_t>();
    SR_CK(cudaEventSynchronize(s->copied[c & 1]));
    memcpy(dst, data + plo, nb);
    for (uint32_t k = 0; k < novl; k++) {
        const uint64_t a = std::max<uint64_t>(ovl[k].start, plo), b = std::min<uint64_t>(ovl[k].start + ovl[k].len, plo + nb);
        if (a < b) memcpy(dst + (a - plo), ovl[k].data + (a - ovl[k].start), b - a);
    }
    return JSGPU_OK;
}

// Chunk c's upload from its slot's pinned buffer on the slot's stream, followed by copied[slot].
static int sr_send(JsSearch* s, const SrChunks& ch, uint64_t c, std::string& err)
{
    const int sl = (int)(c & 1);
    SR_CK(cudaMemcpyAsync(s->buf[sl].p, s->pin[sl].p, ch.bytes(c), cudaMemcpyHostToDevice, s->st[sl]));
    SR_CK(cudaEventRecord(s->copied[sl], s->st[sl]));
    return JSGPU_OK;
}

int js_search_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, const uint8_t* pats, const uint32_t* lens,
                  uint32_t npat, uint64_t* counts, uint32_t* pos, uint64_t cap, std::string& err)
{
    for (uint32_t k = 0; k < npat; k++) counts[k] = 0;
    if (n == 0) return JSGPU_OK;

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
    const SrChunks ch(n, 0, n, P.maxlen - 1, false);          // a match belongs to the chunk it starts in
    SR_TRY(sr_open(ps, device, ch, err));
    JsSearch* s = *ps;
    const uint32_t tiles = (uint32_t)(ch.size / SR_TILE);
    for (int i = 0; i < 2; i++) { SR_CK(s->sum[i].reserve((size_t)tiles * npat * 4)); SR_CK(s->off[i].reserve((size_t)tiles * npat * 4)); }
    SR_CK(s->res.reserve(ch.count * npat * 2 * 4));
    SR_CK(s->pat.reserve(hpat.size()));
    SR_CK(s->hash.reserve(hhash.size() * 4));
    SR_CK(cudaMemcpyAsync(s->pat.p, hpat.data(), hpat.size(), cudaMemcpyHostToDevice, s->st[0]));
    SR_CK(cudaMemcpyAsync(s->hash.p, hhash.data(), hhash.size() * 4, cudaMemcpyHostToDevice, s->st[0]));
    SR_CK(cudaStreamSynchronize(s->st[0]));

    int occ = 0;
    SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_search_tiles<false>, SR_THREADS, 0));
    const uint32_t grid = std::max(1u, std::min<uint32_t>(tiles, (uint32_t)(std::max(occ, 1) * sm_count)));
    SrEmit none; memset(&none, 0, sizeof none);

    // chunk c on slot c & 1: uploaded unless it is still there, summarised, and scanned after chunk c - 1's scan
    uint64_t resident = ~0ull;
    auto run_chunk = [&](uint32_t c, bool emit, const SrEmit& em) -> int {
        const int sl = c & 1;
        if (resident != c) {
            SR_TRY(sr_stage(s, ch, c, data, nullptr, 0, err));
            SR_TRY(sr_send(s, ch, c, err));
            resident = c;
        }
        const uint64_t c0 = ch.first(c), valid = ch.bytes(c);
        const uint32_t nt = (ch.positions(c) + SR_TILE - 1) / SR_TILE;
        const uint8_t* const buf = s->buf[sl].as<uint8_t>();
        uint32_t* const sum = s->sum[sl].as<uint32_t>();
        uint32_t* const off = s->off[sl].as<uint32_t>();
        k_search_tiles<false><<<std::min(grid, nt), SR_THREADS, 0, s->st[sl]>>>(buf, c0, valid, nt, s->pat.as<uint8_t>(),
                                                                                s->hash.as<uint32_t>(), P, sum, nullptr, none, nullptr);
        if (c) SR_CK(cudaStreamWaitEvent(s->st[sl], s->scanned[sl ^ 1], 0));
        k_search_scan<<<npat, 1024, 0, s->st[sl]>>>(sum, nt, off, s->res.as<uint32_t>(), c, npat);
        SR_CK(cudaEventRecord(s->scanned[sl], s->st[sl]));
        if (emit)
            k_search_tiles<true><<<std::min(grid, nt), SR_THREADS, 0, s->st[sl]>>>(buf, c0, valid, nt, s->pat.as<uint8_t>(),
                                                                                   s->hash.as<uint32_t>(), P, sum, off, em,
                                                                                   s->out.as<uint32_t>());
        SR_CK(cudaGetLastError());
        return JSGPU_OK;
    };

    // pass 1: counts per chunk and pattern
    for (uint32_t c = 0; c < ch.count; c++) SR_TRY(run_chunk(c, false, none));
    std::vector<uint32_t> res(ch.count * npat * 2);
    SR_CK(cudaStreamSynchronize(s->st[0])); SR_CK(cudaStreamSynchronize(s->st[1]));
    SR_CK(cudaMemcpy(res.data(), s->res.p, res.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t c = 0; c < ch.count; c++) for (uint32_t k = 0; k < npat; k++) counts[k] += res[2 * ((size_t)c * npat + k)];

    // pass 2: chunks with positions inside `cap`, written in place (pattern k's list follows pattern k-1's)
    if (cap && pos) {
        std::vector<uint64_t> first(npat), run(npat, 0);      // global index of pattern k's first position; its positions before chunk c
        uint64_t acc = 0;
        for (uint32_t k = 0; k < npat; k++) { first[k] = acc; acc += counts[k]; }
        for (uint32_t c = 0; c < ch.count; c++) {
            SrEmit em; memset(&em, 0, sizeof em);
            uint64_t total = 0;
            for (uint32_t k = 0; k < npat; k++) {
                const uint64_t cnt = res[2 * ((size_t)c * npat + k)], g = first[k] + run[k];
                const uint64_t keep = g >= cap ? 0 : std::min<uint64_t>(cnt, cap - g);
                em.lim[k] = (uint32_t)keep; em.base[k] = (uint32_t)total; total += keep;
            }
            if (total) {
                SR_CK(s->out.reserve(total * 4));
                SR_TRY(run_chunk(c, true, em));
                SR_CK(cudaStreamSynchronize(s->st[c & 1]));
                std::vector<uint32_t> h(total);
                SR_CK(cudaMemcpy(h.data(), s->out.p, total * 4, cudaMemcpyDeviceToHost));
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
__global__ void __launch_bounds__(SR_THREADS)
k_find_value(const uint8_t* __restrict__ buf, uint32_t npos, uint32_t pat, uint32_t mask, int forward, uint32_t* __restrict__ res)
{
    __shared__ uint32_t s_best;                              // forward: lowest match, ~0 for none; reverse: highest + 1, 0 for none
    const uint32_t tid = threadIdx.x, lane = tid & 31, none = forward ? 0xFFFFFFFFu : 0u;
    if (tid == 0) s_best = none;
    __syncthreads();
    const uint32_t ntiles = (npos + SR_TILE - 1) / SR_TILE;
    // tiles in search order, so that a CTA can stop at its first tile with a match
    for (uint32_t i = blockIdx.x; i < ntiles; i += gridDim.x) {
        const uint32_t t = forward ? i : ntiles - 1 - i;
        const uint32_t p0 = t * SR_TILE + 16 * tid;
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
        const SrChunks ch(n, (uint64_t)lo, (uint64_t)(hi - lo + 1), len - 1, !forward);   // the halo bytes lie in the file
        SR_TRY(sr_open(ps, device, ch, err));
        JsSearch* s = *ps;
        SR_CK(s->find.reserve(2 * 4));
        SR_CK(s->hfind.reserve(2 * 4));
        uint32_t* const dres = s->find.as<uint32_t>();
        uint32_t* const hres = s->hfind.as<uint32_t>();
        int occ = 0;
        SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_find_value, SR_THREADS, 0));
        const uint32_t grid_max = (uint32_t)(std::max(occ, 1) * sm_count);
        const uint32_t pat = __builtin_bswap32(value) >> (32 - 8 * len);      // the bytes in file order, little-endian
        // The host stages chunk c + 1 while the device searches chunk c; chunk c + 1 goes to the device only if c has no match.
        SR_TRY(sr_stage(s, ch, 0, data, ovl, novl, err));
        for (uint64_t c = 0; c < ch.count; c++) {
            const int sl = (int)(c & 1);
            const uint32_t npos = ch.positions(c);
            SR_TRY(sr_send(s, ch, c, err));
            SR_CK(cudaMemsetAsync(dres + sl, forward ? 0xFF : 0, 4, s->st[sl]));
            const uint32_t grid = std::max(1u, std::min(grid_max, (npos + SR_TILE - 1) / SR_TILE));
            k_find_value<<<grid, SR_THREADS, 0, s->st[sl]>>>(s->buf[sl].as<uint8_t>(), npos, pat, mask, forward, dres + sl);
            SR_CK(cudaGetLastError());
            SR_CK(cudaMemcpyAsync(hres + sl, dres + sl, 4, cudaMemcpyDeviceToHost, s->st[sl]));
            if (c + 1 < ch.count) SR_TRY(sr_stage(s, ch, c + 1, data, ovl, novl, err));
            SR_CK(cudaStreamSynchronize(s->st[sl]));
            const uint32_t r = hres[sl];
            if (forward ? r != 0xFFFFFFFFu : r != 0u) {
                *found = 1; *found_pos = ch.first(c) + (forward ? r : r - 1);
                return JSGPU_OK;
            }
        }
    }
    if (forward) *found = test(*found_pos);                  // the last position, which reads past EOF
    return JSGPU_OK;
}

// ---- every match of a value (jsgpu_find_all) and the extract walk's markers (jsgpu_find_markers), include/jsgpu.h -------
// Each chunk is uploaded once and stays resident while three kernels run on it: k_find_all<false> counts the matches of
// each CTA's run of consecutive tiles, k_find_all_scan turns the counts into output indices from the running total kept on
// the device, and k_find_all<true> writes the positions in file order.  CTA b owns tiles [b * per, (b + 1) * per).
// A search lists one or two match sets over the same chunk: a value (fv_match16) or the scan terminators (fv_term16).

// The PASS-1 scan terminators among positions p0 .. p0 + 15 (p0 a multiple of 16): p with buf[p] == FF and buf[p + 1]
// neither 00 nor D0..D7 (JfifDecode.cpp:5194-5265).  buf holds npos + 1 bytes and is readable as fv_match16's.
__device__ __forceinline__ uint32_t fv_term16(const uint8_t* __restrict__ buf, uint32_t p0, uint32_t npos)
{
    uint32_t m = 0;
    if (p0 < npos) {
        const uint4 a = *(const uint4*)(buf + p0);
        const uint32_t w[5] = {a.x, a.y, a.z, a.w, *(const uint32_t*)(buf + p0 + 16)};
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const uint32_t v = (k % 4) ? __funnelshift_r(w[k / 4], w[k / 4 + 1], 8 * (k % 4)) : w[k / 4];
            const uint32_t b1 = (v >> 8) & 0xFFu;
            if ((v & 0xFFu) == 0xFFu && b1 != 0u && (b1 & 0xF8u) != 0xD0u) m |= 1u << k;
        }
        if (npos - p0 < 16) m &= (1u << (npos - p0)) - 1u;
    }
    return m;
}

// One match set of a chunk: the value pat / mask at positions 0 .. npos - 1, or the terminators there when `term`; the
// positions go to out, at most cap of them in all.
struct FaSet { uint32_t npos, pat, mask, term; uint32_t* out; uint64_t cap; };
struct FaSets { FaSet s[2]; };

__device__ __forceinline__ uint32_t fa_match16(const uint8_t* __restrict__ buf, uint32_t p0, const FaSet& f)
{
    return f.term ? fv_term16(buf, p0, f.npos) : fv_match16(buf, p0, f.npos, f.pat, f.mask);
}

template <bool EMIT, int NSET>
__global__ void __launch_bounds__(SR_THREADS)
k_find_all(const uint8_t* __restrict__ buf, uint32_t npos, FaSets sets, uint32_t per, uint32_t chunk_pos,
           uint32_t* __restrict__ cta /*[NSET][2][gridDim.x]: counts, then first output index*/)
{
    __shared__ uint32_t s_w[SR_THREADS / 32 + 1];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t ntiles = (npos + SR_TILE - 1) / SR_TILE;
    const uint32_t t0 = blockIdx.x * per, t1 = min(ntiles, t0 + per);
#pragma unroll
    for (int k = 0; k < NSET; k++) {
        const FaSet& f = sets.s[k];
        uint32_t* const ck = cta + 2 * gridDim.x * k;
        if (!EMIT) {
            uint32_t c = 0;
            for (uint32_t t = t0; t < t1; t++) c += __popc(fa_match16(buf, t * SR_TILE + 16 * tid, f));
            c = __reduce_add_sync(0xffffffffu, c);
            if (lane == 0) s_w[warp] = c;
            __syncthreads();
            if (tid == 0) {
                uint32_t sum = 0;
                for (int w = 0; w < SR_THREADS / 32; w++) sum += s_w[w];
                ck[blockIdx.x] = sum;
            }
            __syncthreads();
            continue;
        }
        uint32_t j = ck[gridDim.x + blockIdx.x];             // this CTA's first output index
        if (ck[blockIdx.x] == 0 || j >= f.cap) continue;
        for (uint32_t t = t0; t < t1 && j < f.cap; t++) {
            uint32_t m = fa_match16(buf, t * SR_TILE + 16 * tid, f);
            uint64_t o = js_block_scan<SR_THREADS>((uint32_t)__popc(m), 0u, js_add, j, s_w);   // advances j past the tile
            const uint32_t p = chunk_pos + t * SR_TILE + 16 * tid;
            while (m && o < f.cap) { f.out[o++] = p + (uint32_t)__ffs((int)m) - 1; m &= m - 1; }
        }
    }
}

// CTA k: the first output index of every CTA of the chunk in set k, from set k's running total, which it then advances.
__global__ void __launch_bounds__(1024)
k_find_all_scan(uint32_t* __restrict__ cta, uint32_t ncta, uint32_t* __restrict__ total)
{
    __shared__ uint32_t s_w[33];
    cta += 2 * ncta * blockIdx.x; total += blockIdx.x;
    uint32_t run = *total;
    for (uint32_t b0 = 0; b0 < ncta; b0 += 1024) {
        const uint32_t b = b0 + threadIdx.x;
        const uint32_t o = js_block_scan<1024>(b < ncta ? cta[b] : 0u, 0u, js_add, run, s_w);
        if (b < ncta) cta[ncta + b] = o;
    }
    if (threadIdx.x == 0) *total = run;
}

// One streaming pass of NSET match sets over positions 0 .. npos - 1 of the file, chunks carrying `halo` bytes.  set(k, plo,
// cnpos) gives set k's FaSet for the chunk of cnpos positions from plo (npos, pat, mask, term); counts[k] receive complete
// counts and pos[k] at most caps[k] positions.
template <int NSET, typename SetOf>
static int fa_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, uint64_t npos, uint32_t halo,
                  const jsgpu_overlay* ovl, uint32_t novl, SetOf set, uint64_t* counts, uint32_t* const* pos, const uint64_t* caps,
                  std::string& err)
{
    for (int k = 0; k < NSET; k++) counts[k] = 0;
    if (!npos) return JSGPU_OK;
    const SrChunks ch(n, 0, npos, halo, false);
    SR_TRY(sr_open(ps, device, ch, err));
    JsSearch* s = *ps;
    int occ = 0;
    SR_CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_find_all<true, NSET>, SR_THREADS, 0));
    const uint32_t grid_max = (uint32_t)(std::max(occ, 1) * sm_count);
    for (int i = 0; i < 2; i++) SR_CK(s->cta[i].reserve(2 * NSET * (size_t)grid_max * 4));
    uint64_t keep[NSET], off[NSET], all = 0;                  // positions each device list can hold, and where it starts
    for (int k = 0; k < NSET; k++) { keep[k] = std::min<uint64_t>(caps[k], ch.npos); off[k] = all; all += keep[k]; }
    if (all) SR_CK(s->out.reserve(all * 4));
    SR_CK(s->total.reserve(4 * NSET));
    uint32_t* const total = s->total.as<uint32_t>();
    SR_CK(cudaMemsetAsync(total, 0, 4 * NSET, s->st[0]));
    SR_CK(cudaEventRecord(s->scanned[1], s->st[0]));                      // chunk 0's scan follows the reset

    bool emit = false;
    for (int k = 0; k < NSET; k++) emit |= keep[k] != 0;
    for (uint64_t c = 0; c < ch.count; c++) {
        const int sl = (int)(c & 1);
        const uint32_t cnpos = ch.positions(c), plo = (uint32_t)ch.first(c);
        SR_TRY(sr_stage(s, ch, c, data, ovl, novl, err));
        SR_TRY(sr_send(s, ch, c, err));
        const uint8_t* const buf = s->buf[sl].as<uint8_t>();
        uint32_t* const cta = s->cta[sl].as<uint32_t>();
        FaSets sets = {};
        for (int k = 0; k < NSET; k++) {
            sets.s[k] = set(k, plo, cnpos);
            sets.s[k].out = s->out.as<uint32_t>() + off[k];
            sets.s[k].cap = keep[k];
        }
        const uint32_t ntiles = (cnpos + SR_TILE - 1) / SR_TILE;
        const uint32_t grid = std::max(1u, std::min(grid_max, ntiles)), per = (ntiles + grid - 1) / grid;
        k_find_all<false, NSET><<<grid, SR_THREADS, 0, s->st[sl]>>>(buf, cnpos, sets, per, plo, cta);
        SR_CK(cudaStreamWaitEvent(s->st[sl], s->scanned[sl ^ 1], 0));  // the previous chunk has advanced the totals
        k_find_all_scan<<<NSET, 1024, 0, s->st[sl]>>>(cta, grid, total);
        SR_CK(cudaEventRecord(s->scanned[sl], s->st[sl]));
        if (emit) k_find_all<true, NSET><<<grid, SR_THREADS, 0, s->st[sl]>>>(buf, cnpos, sets, per, plo, cta);
        SR_CK(cudaGetLastError());
    }
    SR_CK(cudaStreamSynchronize(s->st[0])); SR_CK(cudaStreamSynchronize(s->st[1]));
    uint32_t tot[NSET];
    SR_CK(cudaMemcpy(tot, total, 4 * NSET, cudaMemcpyDeviceToHost));
    for (int k = 0; k < NSET; k++) {
        counts[k] = tot[k];
        const uint64_t got = std::min<uint64_t>(tot[k], keep[k]);
        if (got) SR_CK(cudaMemcpy(pos[k], s->out.as<uint32_t>() + off[k], got * 4, cudaMemcpyDeviceToHost));
    }
    return JSGPU_OK;
}

int js_find_all_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, uint32_t value, uint32_t len,
                    uint64_t* count, uint32_t* pos, uint64_t cap, std::string& err)
{
    *count = 0;
    const uint32_t mask = len == 4 ? 0xFFFFFFFFu : (1u << (8 * len)) - 1u;
    if (n < len || (value & ~mask)) return JSGPU_OK;         // no position, or a value wider than len bytes
    const uint32_t pat = __builtin_bswap32(value) >> (32 - 8 * len);      // the bytes in file order, little-endian
    auto set = [&](int, uint32_t, uint32_t cnpos) { return FaSet{cnpos, pat, mask, 0u, nullptr, 0}; };
    return fa_run<1>(ps, device, sm_count, data, n, n - len + 1, len - 1, nullptr, 0, set, count, &pos, &cap, err);
}

// Set 0: FF D8 FF at 0 .. n - 3; set 1: the terminators at 0 .. n - 2 (an FF in the last byte is followed by 0, the byte
// Buf() reads past the end of the file, so it ends nothing).  Chunks cover the terminator positions with 2 halo bytes.
int js_find_markers_run(JsSearch** ps, int device, int sm_count, const uint8_t* data, uint64_t n, const jsgpu_overlay* ovl,
                        uint32_t novl, uint32_t* soi_pos, uint64_t soi_cap, uint64_t* nsoi, uint32_t* term_pos, uint64_t term_cap,
                        uint64_t* nterm, std::string& err)
{
    *nsoi = *nterm = 0;
    if (n < 2) return JSGPU_OK;
    const uint64_t nsoi_pos = n >= 3 ? n - 2 : 0;
    auto set = [&](int k, uint32_t plo, uint32_t cnpos) {
        if (k == 1) return FaSet{cnpos, 0u, 0u, 1u, nullptr, 0};
        const uint32_t np = plo < nsoi_pos ? (uint32_t)std::min<uint64_t>(cnpos, nsoi_pos - plo) : 0u;
        return FaSet{np, 0xFFD8FFu, 0xFFFFFFu, 0u, nullptr, 0};           // FF D8 FF read little-endian is FF D8 FF
    };
    uint64_t counts[2];
    uint32_t* const pos[2] = {soi_pos, term_pos};
    const uint64_t caps[2] = {soi_cap, term_cap};
    SR_TRY(fa_run<2>(ps, device, sm_count, data, n, n - 1, 2, ovl, novl, set, counts, pos, caps, err));
    *nsoi = counts[0]; *nterm = counts[1];
    return JSGPU_OK;
}
