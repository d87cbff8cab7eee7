// synth_jpeg.cpp — seeded synthetic baseline-JPEG generator (bench / test INPUT tool; host only).
//
// Produces restart-segmented baseline JPEG files of the kind BASELINE.json's configs name
// (SURVEY.md §8d): SOF0, 8-bit, 3 components (ids 1,2,3; or 1 for grayscale), one interleaved scan,
// Annex-K Huffman tables or per-image optimised ones, IJG-scaled Annex-K quantisation at a given
// quality, DRI = any MCU count.  Pixel content: smooth sinusoid field + zero-mean noise of
// standard deviation 12 per channel (Irwin-Hall(4) noise from a splitmix64 stream: bounded,
// near-Gaussian, bit-reproducible everywhere).  Everything here is written for this repo;
// tables are the published ITU-T T.81 Annex K values.
#include <cstdint>
#include <cstring>
#include <cmath>
#include <vector>
#include <thread>
#include <atomic>
#include <algorithm>
#include "../annex_k.h"

namespace {

const uint8_t kZigZag[64] = {
     0, 1, 8,16, 9, 2, 3,10, 17,24,32,25,18,11, 4, 5, 12,19,26,33,40,48,41,34, 27,20,13, 6, 7,14,21,28,
    35,42,49,56,57,50,43,36, 29,22,15,23,30,37,44,51, 58,59,52,45,38,31,39,46, 53,60,61,54,47,55,62,63 };

// T.81 Table K.1 / K.2 (natural order)
const uint8_t kQLum[64] = {
    16,11,10,16,24,40,51,61, 12,12,14,19,26,58,60,55, 14,13,16,24,40,57,69,56, 14,17,22,29,51,87,80,62,
    18,22,37,56,68,109,103,77, 24,35,55,64,81,104,113,92, 49,64,78,87,103,121,120,101, 72,92,95,98,112,100,103,99 };
const uint8_t kQChr[64] = {
    17,18,24,47,99,99,99,99, 18,21,26,66,99,99,99,99, 24,26,56,99,99,99,99,99, 47,66,99,99,99,99,99,99,
    99,99,99,99,99,99,99,99, 99,99,99,99,99,99,99,99, 99,99,99,99,99,99,99,99, 99,99,99,99,99,99,99,99 };
// T.81 Tables K.3-K.6 (BITS, HUFFVAL) come from annex_k.h
using namespace annex_k;

struct HuffSpec { uint8_t bits[16]; uint8_t vals[256]; int nvals; };
struct HuffEnc { uint16_t code[256]; uint8_t len[256]; };

void make_enc(const HuffSpec& s, HuffEnc& e)
{
    memset(&e, 0, sizeof e);
    unsigned code = 0, k = 0;
    for (int l = 1; l <= 16; l++) { for (int i = 0; i < s.bits[l - 1]; i++) { e.code[s.vals[k]] = (uint16_t)code; e.len[s.vals[k]] = (uint8_t)l; code++; k++; } code <<= 1; }
}

// Length-limited Huffman table from symbol frequencies (procedure of T.81 Annex K.2, Figures
// K.1-K.4: code-size computation with a reserved all-ones code point, then limiting to 16 bits).
void optimal_spec(const long* freq_in, HuffSpec& s)
{
    long freq[257]; int codesize[257], others[257];
    for (int i = 0; i < 256; i++) freq[i] = freq_in[i];
    freq[256] = 1;
    memset(codesize, 0, sizeof codesize);
    for (int i = 0; i < 257; i++) others[i] = -1;
    for (;;) {
        int c1 = -1, c2 = -1; long v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = 1000000000L;
        for (int i = 0; i <= 256; i++) if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
        if (c2 < 0) break;
        freq[c1] += freq[c2]; freq[c2] = 0;
        codesize[c1]++; while (others[c1] >= 0) { c1 = others[c1]; codesize[c1]++; }
        others[c1] = c2;
        codesize[c2]++; while (others[c2] >= 0) { c2 = others[c2]; codesize[c2]++; }
    }
    int bits[40]; memset(bits, 0, sizeof bits);
    for (int i = 0; i <= 256; i++) if (codesize[i]) bits[codesize[i] > 39 ? 39 : codesize[i]]++;
    for (int i = 39; i > 16; i--) {
        while (bits[i] > 0) {
            int j = i - 2; while (bits[j] == 0) j--;
            bits[i] -= 2; bits[i - 1]++; bits[j + 1] += 2; bits[j]--;
        }
    }
    int i = 16; while (bits[i] == 0) i--;
    bits[i]--;                                            // remove the reserved code point
    for (int l = 1; l <= 16; l++) s.bits[l - 1] = (uint8_t)bits[l];
    int k = 0;
    for (int l = 1; l <= 32; l++) for (int j = 0; j < 256; j++) if (codesize[j] == l) s.vals[k++] = (uint8_t)j;
    s.nvals = k;
}

struct BitWriter {
    std::vector<uint8_t>& out; uint64_t acc = 0; int n = 0;
    explicit BitWriter(std::vector<uint8_t>& o) : out(o) {}
    inline void put(unsigned code, int len) {
        acc = (acc << len) | (code & ((1u << len) - 1)); n += len;
        while (n >= 8) { uint8_t b = (uint8_t)(acc >> (n - 8)); out.push_back(b); if (b == 0xFF) out.push_back(0); n -= 8; }
    }
    inline void flush() { if (n > 0) put((1u << (8 - n)) - 1, 8 - n); acc = 0; n = 0; }    // pad with 1-bits
};

inline uint64_t splitmix(uint64_t& s) { uint64_t z = (s += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
// Irwin-Hall(4) from one 64-bit draw, scaled to standard deviation 12: sum of four U[0,65535]
inline float noise12(uint64_t& s)
{
    uint64_t r = splitmix(s);
    int sum = (int)(r & 0xFFFF) + (int)((r >> 16) & 0xFFFF) + (int)((r >> 32) & 0xFFFF) + (int)(r >> 48);
    // mean 2*65535, variance 4*(65536^2-1)/12 -> sd = 37837.2
    return (float)(sum - 131070) * (12.0f / 37837.2f);
}

void fdct8x8(const float* in, float* out, const float (*C)[8])
{
    float tmp[64];
    for (int y = 0; y < 8; y++) for (int u = 0; u < 8; u++) { float s = 0; for (int x = 0; x < 8; x++) s += in[y * 8 + x] * C[u][x]; tmp[y * 8 + u] = s; }
    for (int v = 0; v < 8; v++) for (int u = 0; u < 8; u++) { float s = 0; for (int y = 0; y < 8; y++) s += tmp[y * 8 + u] * C[v][y]; out[v * 8 + u] = s; }
}

inline int bitsize(int v) { int a = v < 0 ? -v : v, n = 0; while (a) { n++; a >>= 1; } return n; }

struct Params { int w, h, subs, quality, ri, optimize; uint64_t seed; };

void put16(std::vector<uint8_t>& o, unsigned v) { o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }

void encode_one(const Params& p, std::vector<uint8_t>& out)
{
    const int ncomp = (p.subs == 3) ? 1 : 3;
    const int H0 = (p.subs == 1 || p.subs == 2) ? 2 : 1, V0 = (p.subs == 2) ? 2 : 1;
    const int mcuw = 8 * H0, mcuh = 8 * V0;
    const int mx = (p.w + mcuw - 1) / mcuw, my = (p.h + mcuh - 1) / mcuh;
    const int W = mx * mcuw, Hh = my * mcuh;
    // ---- pixels -> YCbCr planes (padded by edge replication of coordinates) --------------------
    std::vector<float> Y((size_t)W * Hh), Cb, Cr;
    if (ncomp == 3) { Cb.resize((size_t)W * Hh); Cr.resize((size_t)W * Hh); }
    std::vector<float> sx37(W), sx11(W), cy23(Hh), cy17(Hh);
    for (int x = 0; x < W; x++) { int xx = std::min(x, p.w - 1); sx37[x] = sinf(xx / 37.0f); sx11[x] = xx / 11.0f; }
    for (int y = 0; y < Hh; y++) { int yy = std::min(y, p.h - 1); cy23[y] = cosf(yy / 23.0f); cy17[y] = cosf(yy / 17.0f); }
    for (int y = 0; y < Hh; y++) {
        const int yy = std::min(y, p.h - 1);
        uint64_t rs = p.seed * 0x9E3779B97F4A7C15ull + (uint64_t)yy * 0xD1B54A32D192ED03ull + 0x1234567;
        // noise is a function of (seed, source row, source column) so padding replicates real pixels
        std::vector<float> nz((size_t)p.w * 3);
        for (int x = 0; x < p.w * 3; x++) nz[x] = noise12(rs);
        const float g2 = 60.0f, ph = yy / 50.0f;
        for (int x = 0; x < W; x++) {
            const int xx = std::min(x, p.w - 1);
            float r = 128.0f + 80.0f * sx37[x] * cy23[y] + nz[xx * 3 + 0];
            float g = 128.0f + g2 * sinf(sx11[x] + ph) + nz[xx * 3 + 1];
            float b = 128.0f + 70.0f * cy17[y] + nz[xx * 3 + 2];
            r = std::min(255.0f, std::max(0.0f, floorf(r))); g = std::min(255.0f, std::max(0.0f, floorf(g))); b = std::min(255.0f, std::max(0.0f, floorf(b)));
            if (ncomp == 1) { Y[(size_t)y * W + x] = r - 128.0f; }
            else {
                Y [(size_t)y * W + x] = 0.299f * r + 0.587f * g + 0.114f * b - 128.0f;
                Cb[(size_t)y * W + x] = -0.168736f * r - 0.331264f * g + 0.5f * b;
                Cr[(size_t)y * W + x] = 0.5f * r - 0.418688f * g - 0.081312f * b;
            }
        }
    }
    // ---- quantisation tables (IJG quality scaling) ------------------------------------------------
    int q = std::min(100, std::max(1, p.quality));
    int scale = q < 50 ? 5000 / q : 200 - 2 * q;
    uint16_t QT[2][64];
    for (int t = 0; t < 2; t++) for (int i = 0; i < 64; i++) { int v = ((t ? kQChr[i] : kQLum[i]) * scale + 50) / 100; QT[t][i] = (uint16_t)std::min(255, std::max(1, v)); }
    // ---- DCT + quantise: coefficient blocks in scan (MCU) order, zig-zag order inside -------------
    float C[8][8];
    for (int u = 0; u < 8; u++) for (int x = 0; x < 8; x++) C[u][x] = (u == 0 ? 0.35355339f : 0.5f) * cosf((2 * x + 1) * u * 3.14159265358979f / 16.0f);
    struct CompInfo { int H, V, tq; const std::vector<float>* plane; } ci[3];
    ci[0] = {H0, V0, 0, &Y}; if (ncomp == 3) { ci[1] = {1, 1, 1, &Cb}; ci[2] = {1, 1, 1, &Cr}; }
    int bpm = 0; for (int c = 0; c < ncomp; c++) bpm += ci[c].H * ci[c].V;
    const size_t nmcu = (size_t)mx * my;
    std::vector<int16_t> coefs(nmcu * bpm * 64);
    {
        size_t bi = 0; float blk[64], dct[64];
        for (int myi = 0; myi < my; myi++) for (int mxi = 0; mxi < mx; mxi++) for (int c = 0; c < ncomp; c++) {
            const int eh = H0 / ci[c].H, ev = V0 / ci[c].V;
            for (int v = 0; v < ci[c].V; v++) for (int h = 0; h < ci[c].H; h++) {
                const int x0 = mxi * mcuw + h * 8 * eh, y0 = myi * mcuh + v * 8 * ev;
                for (int y = 0; y < 8; y++) for (int x = 0; x < 8; x++) {
                    float s = 0;
                    for (int dy = 0; dy < ev; dy++) for (int dx = 0; dx < eh; dx++) s += (*ci[c].plane)[(size_t)(y0 + y * ev + dy) * W + (x0 + x * eh + dx)];
                    blk[y * 8 + x] = s / (float)(eh * ev);
                }
                fdct8x8(blk, dct, C);
                int16_t* o = &coefs[bi * 64];
                for (int k = 0; k < 64; k++) { float f = dct[kZigZag[k]] / (float)QT[ci[c].tq][kZigZag[k]]; o[k] = (int16_t)lrintf(f); }
                bi++;
            }
        }
    }
    // ---- Huffman tables -----------------------------------------------------------------------
    HuffSpec spec[2][2];       // [class][table]
    auto setspec = [](HuffSpec& s, const uint8_t* bits, const uint8_t* vals, int n) { memcpy(s.bits, bits, 16); memcpy(s.vals, vals, n); s.nvals = n; };
    setspec(spec[0][0], kDcLumBits, kDcVals, 12); setspec(spec[0][1], kDcChrBits, kDcVals, 12);
    setspec(spec[1][0], kAcLumBits, kAcLumVals, 162); setspec(spec[1][1], kAcChrBits, kAcChrVals, 162);
    const int ri = p.ri > 0 ? p.ri : 0;
    if (p.optimize) {
        long fr[2][2][256]; memset(fr, 0, sizeof fr);
        size_t bi = 0; int pred[3] = {0, 0, 0};
        for (size_t m = 0; m < nmcu; m++) {
            if (ri && m % ri == 0) pred[0] = pred[1] = pred[2] = 0;
            for (int c = 0; c < ncomp; c++) for (int b = 0; b < ci[c].H * ci[c].V; b++, bi++) {
                const int16_t* o = &coefs[bi * 64]; int t = ci[c].tq;
                int d = o[0] - pred[c]; pred[c] = o[0]; fr[0][t][bitsize(d)]++;
                int run = 0;
                for (int k = 1; k < 64; k++) { if (o[k] == 0) { run++; continue; } while (run > 15) { fr[1][t][0xF0]++; run -= 16; } fr[1][t][(run << 4) | bitsize(o[k])]++; run = 0; }
                if (run) fr[1][t][0]++;
            }
        }
        for (int cl = 0; cl < 2; cl++) for (int t = 0; t < (ncomp == 3 ? 2 : 1); t++) optimal_spec(fr[cl][t], spec[cl][t]);
    }
    HuffEnc enc[2][2];
    for (int cl = 0; cl < 2; cl++) for (int t = 0; t < 2; t++) make_enc(spec[cl][t], enc[cl][t]);
    // ---- headers --------------------------------------------------------------------------------
    out.clear(); out.reserve(nmcu * bpm * 24 + 1024);
    out.push_back(0xFF); out.push_back(0xD8);
    const uint8_t app0[] = {0xFF,0xE0,0,16,'J','F','I','F',0,1,1,0,0,1,0,1,0,0}; out.insert(out.end(), app0, app0 + sizeof app0);
    for (int t = 0; t < (ncomp == 3 ? 2 : 1); t++) { out.push_back(0xFF); out.push_back(0xDB); put16(out, 67); out.push_back((uint8_t)t); for (int k = 0; k < 64; k++) out.push_back((uint8_t)QT[t][kZigZag[k]]); }
    out.push_back(0xFF); out.push_back(0xC0); put16(out, 8 + 3 * ncomp); out.push_back(8); put16(out, p.h); put16(out, p.w); out.push_back((uint8_t)ncomp);
    for (int c = 0; c < ncomp; c++) { out.push_back((uint8_t)(c + 1)); out.push_back((uint8_t)((ci[c].H << 4) | ci[c].V)); out.push_back((uint8_t)ci[c].tq); }
    for (int t = 0; t < (ncomp == 3 ? 2 : 1); t++) for (int cl = 0; cl < 2; cl++) {
        const HuffSpec& s = spec[cl][t];
        out.push_back(0xFF); out.push_back(0xC4); put16(out, 2 + 1 + 16 + s.nvals); out.push_back((uint8_t)((cl << 4) | t));
        out.insert(out.end(), s.bits, s.bits + 16); out.insert(out.end(), s.vals, s.vals + s.nvals);
    }
    if (ri) { out.push_back(0xFF); out.push_back(0xDD); put16(out, 4); put16(out, ri); }
    out.push_back(0xFF); out.push_back(0xDA); put16(out, 6 + 2 * ncomp); out.push_back((uint8_t)ncomp);
    for (int c = 0; c < ncomp; c++) { out.push_back((uint8_t)(c + 1)); out.push_back((uint8_t)((ci[c].tq << 4) | ci[c].tq)); }
    out.push_back(0); out.push_back(63); out.push_back(0);
    // ---- entropy-coded data ---------------------------------------------------------------------
    BitWriter bw(out);
    size_t bi = 0; int pred[3] = {0, 0, 0}; int rstn = 0;
    for (size_t m = 0; m < nmcu; m++) {
        if (ri && m > 0 && m % ri == 0) { bw.flush(); out.push_back(0xFF); out.push_back((uint8_t)(0xD0 + (rstn & 7))); rstn++; pred[0] = pred[1] = pred[2] = 0; }
        for (int c = 0; c < ncomp; c++) for (int b = 0; b < ci[c].H * ci[c].V; b++, bi++) {
            const int16_t* o = &coefs[bi * 64]; const int t = ci[c].tq;
            int d = o[0] - pred[c]; pred[c] = o[0];
            int s = bitsize(d);
            bw.put(enc[0][t].code[s], enc[0][t].len[s]);
            if (s) bw.put((unsigned)(d < 0 ? d - 1 : d), s);
            int run = 0;
            for (int k = 1; k < 64; k++) {
                int v = o[k];
                if (v == 0) { run++; continue; }
                while (run > 15) { bw.put(enc[1][t].code[0xF0], enc[1][t].len[0xF0]); run -= 16; }
                int sz = bitsize(v); int sym = (run << 4) | sz;
                bw.put(enc[1][t].code[sym], enc[1][t].len[sym]);
                bw.put((unsigned)(v < 0 ? v - 1 : v), sz);
                run = 0;
            }
            if (run) bw.put(enc[1][t].code[0], enc[1][t].len[0]);
        }
    }
    bw.flush();
    out.push_back(0xFF); out.push_back(0xD9);
}

} // namespace

extern "C" {

// Encode one image; returns bytes written, or -(needed bytes) when out_cap is too small.
// subsampling: 0 = 4:4:4, 1 = 4:2:2 (2x1), 2 = 4:2:0 (2x2), 3 = grayscale.  restart_interval in MCUs (0 = no DRI).
long long jssynth_encode(int width, int height, int subsampling, int quality, int restart_interval, int optimize,
                         unsigned long long seed, unsigned char* out, unsigned long long out_cap)
{
    if (width <= 0 || height <= 0 || width > 65535 || height > 65535 || subsampling < 0 || subsampling > 3) return 0;
    Params p{width, height, subsampling, quality, restart_interval, optimize, seed};
    std::vector<uint8_t> v; encode_one(p, v);
    if (v.size() > out_cap) return -(long long)v.size();
    memcpy(out, v.data(), v.size());
    return (long long)v.size();
}

// Encode n images with per-image parameter arrays on `threads` host threads into one buffer;
// offsets[n+1] receives the byte offsets.  Returns total bytes or -(needed) if the buffer is too small.
long long jssynth_encode_batch(int n, const int* width, const int* height, const int* subsampling, const int* quality,
                               const int* restart_interval, const int* optimize, const unsigned long long* seed,
                               int threads, unsigned char* out, unsigned long long out_cap, unsigned long long* offsets)
{
    if (n <= 0) return 0;
    if (threads < 1) threads = 1;
    std::vector<std::vector<uint8_t>> bufs((size_t)n);
    std::atomic<int> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < threads; t++) th.emplace_back([&] {
        for (;;) { int i = next.fetch_add(1); if (i >= n) break;
            Params p{width[i], height[i], subsampling[i], quality[i], restart_interval[i], optimize[i], seed[i]};
            encode_one(p, bufs[(size_t)i]); }
    });
    for (auto& x : th) x.join();
    unsigned long long tot = 0;
    for (int i = 0; i < n; i++) { offsets[i] = tot; tot += bufs[(size_t)i].size(); }
    offsets[n] = tot;
    if (tot > out_cap) return -(long long)tot;
    for (int i = 0; i < n; i++) memcpy(out + offsets[i], bufs[(size_t)i].data(), bufs[(size_t)i].size());
    return (long long)tot;
}

}
