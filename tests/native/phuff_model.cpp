// TEST INFRASTRUCTURE (never linked into libjsgpu.so): host model of the self-synchronising Huffman passes.
//
// It compiles the SAME per-slot code the CUDA kernels run (jpegsnoop_b200/csrc/jsgpu_phuff_core.cuh: ph_run,
// ph_guess_slot, ph_fix_slot, ph_vseg) with g++, executes the passes slot by slot on the CPU in a chosen order
// (descending = every slot sees its predecessor's state of the PREVIOUS round, like concurrent GPU threads; ascending;
// pseudo-random), and checks the virtual restart intervals they produce against a plain sequential walk of the scan
// written here independently: every virtual interval must start at the true bit position of the MCU it claims, with the
// true DC predictors, and the intervals must tile the MCUs of every real interval.  No pixels are produced here —
// this checks the host-testable half of the GPU path, not a decode.
#include "../../jpegsnoop_b200/csrc/jsgpu_tables_host.h"
#include "../../jpegsnoop_b200/csrc/jsgpu_phuff_core.cuh"
#include <vector>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <algorithm>

namespace {

struct Geo { uint32_t ns, bpm, ri, nmcu, nseg, H[3], V[3], sdc[3], sac[3], dqt[3], pshift; };

bool make_geo(const jsgpu_image_desc& d, Geo& g)
{
    memset(&g, 0, sizeof g);
    g.ns = d.num_sos_comps;
    if (g.ns != 1 && g.ns != 3) return false;
    uint32_t hmax = 0, vmax = 0;
    for (uint32_t c = 0; c < g.ns; c++) { g.H[c] = d.samp_h[c]; g.V[c] = d.samp_v[c]; hmax = std::max(hmax, g.H[c]); vmax = std::max(vmax, g.V[c]); }
    if (g.ns == 1) { g.H[0] = g.V[0] = 1; hmax = vmax = 1; }
    if (!hmax || !vmax) return false;
    const uint32_t mw = hmax * 8, mh = vmax * 8;
    const uint32_t mx = (d.dim_x + mw - 1) / mw, my = (d.dim_y + mh - 1) / mh;
    g.nmcu = mx * my;
    for (uint32_t c = 0; c < g.ns; c++) { g.bpm += g.H[c] * g.V[c]; g.sdc[c] = d.dht_dc_sel[c]; g.sac[c] = 4 + d.dht_ac_sel[c]; g.dqt[c] = d.dqt_sel[c]; }
    g.ri = (d.restart_en && d.restart_interval) ? d.restart_interval : g.nmcu;
    g.nseg = (g.nmcu + g.ri - 1) / g.ri;
    g.pshift = d.precision > 8 ? d.precision - 8 : 0;
    return true;
}

struct Interval { uint32_t s0, ulen; unsigned long long uoff; };

// marker walk + FF00 unstuffing on the host, into the layout k_unstuff produces (big-endian words, 16-byte aligned
// copies at (s0 & ~15) + JS_USLACK*k, 16 bytes of 0xFF behind each)
void unstuff(const uint8_t* scan, uint64_t n, const Geo& g, std::vector<Interval>& iv, std::vector<uint8_t>& ub)
{
    iv.assign(g.nseg, Interval{0, 0, 0});
    ub.assign(n + (uint64_t)JS_USLACK * g.nseg + 128 + 16384, 0xFF);
    std::vector<uint32_t> st(g.nseg, 0), en(g.nseg, 0);
    uint32_t k = 0, endpos = (uint32_t)n;
    for (uint64_t q = 0; q + 1 < n; q++) {
        if (scan[q] != 0xFF) continue;
        const uint8_t m = scan[q + 1];
        if (m >= 0xD0 && m <= 0xD7) { if (k < g.nseg) en[k] = (uint32_t)q; if (k + 1 < g.nseg) st[k + 1] = (uint32_t)q + 2; k++; q++; }
        else if (m != 0x00 && m != 0xFF) { endpos = (uint32_t)q; break; }
    }
    const uint32_t nf = k + 1;
    if (nf <= g.nseg) en[nf - 1] = endpos;
    for (uint32_t j = nf; j < g.nseg; j++) st[j] = en[j] = endpos;
    for (uint32_t j = 0; j < g.nseg; j++) {
        Interval& I = iv[j]; I.s0 = st[j];
        I.uoff = (unsigned long long)(st[j] & ~15u) + (unsigned long long)JS_USLACK * j;
        std::vector<uint8_t> out;
        for (uint32_t q = st[j]; q < en[j]; q++) {
            if (scan[q] == 0 && q > st[j] && scan[q - 1] == 0xFF) continue;
            out.push_back(scan[q]);
        }
        I.ulen = (uint32_t)out.size();
        out.resize((out.size() + 16 + 3) & ~3ull, 0xFF);
        for (size_t w = 0; w < out.size() / 4; w++)            // store as big-endian words
            for (int b2 = 0; b2 < 4; b2++) ub[I.uoff + w * 4 + b2] = out[w * 4 + 3 - b2];
    }
}

struct Truth { std::vector<uint32_t> mcu_bit; std::vector<int16_t> dc; uint32_t nmcu_done; bool dead; };   // per interval

uint32_t peek(const uint32_t* w, uint32_t bp)
{
    const uint32_t i = bp >> 5, s = bp & 31;
    return s ? ((w[i] << s) | (w[i + 1] >> (32 - s))) : w[i];
}
uint32_t lookup(const DevTableSet& ts, uint32_t slot, uint32_t top)
{
    uint32_t e = ts.lut[slot][top >> (32 - JS_LUT_BITS)];
    if (e & 0x8000) e = ts.lut2[slot][(e & 0x7FFF) + ((top >> 16) & ((1u << JS_LUT2_BITS) - 1))];
    return e;
}
// plain sequential walk of one interval: bit position and DC predictors at every MCU start
void walk(const DevTableSet& ts, const Geo& g, const uint32_t* w, uint32_t ulen, uint32_t cnt, Truth& t)
{
    t.mcu_bit.clear(); t.dc.clear(); t.dead = false;
    uint32_t bp = 0; int16_t dc[3] = {0, 0, 0};
    for (uint32_t m = 0; m < cnt; m++) {
        if (bp >= ulen * 8u) break;
        t.mcu_bit.push_back(bp); t.dc.push_back(dc[0]); t.dc.push_back(dc[1]); t.dc.push_back(dc[2]);
        for (uint32_t c = 0; c < g.ns && !t.dead; c++)
            for (uint32_t bi = 0; bi < g.H[c] * g.V[c] && !t.dead; bi++) {
                uint32_t e = lookup(ts, g.sdc[c], peek(w, bp));
                if (!e) { t.dead = true; break; }
                bp += e >> 8;
                uint32_t size = e & 15, run = (e >> 4) & 15;
                uint32_t tv = peek(w, bp);
                int val = size ? (int)(tv >> (32 - size)) : 0;
                if (size && !(tv >> 31)) val -= (int)((1u << size) - 1);
                if (g.pshift) val /= (1 << g.pshift);
                bp += size;
                const uint32_t q = ts.qz[g.dqt[c]][run];
                if ((q >> 16) == 0) dc[c] = (int16_t)(dc[c] + (int16_t)(val * (int)(q & 0xFFFF)));
                uint32_t pos = 1 + run;
                while (pos < 64) {
                    e = lookup(ts, g.sac[c], peek(w, bp));
                    if (!e) { t.dead = true; break; }
                    bp += (e >> 8) + (e & 15);
                    if ((e & 0xFF) == 0) break;
                    pos += ((e >> 4) & 15) + 1;
                }
            }
        if (t.dead) break;
    }
    t.nmcu_done = (uint32_t)t.mcu_bit.size();
}

}  // namespace

// Every interval's MCU start bits and DC predictors by the sequential walk, concatenated (at most cap MCUs); ulen[k] =
// unstuffed length of interval k in bytes (at most nseg_cap intervals).  Returns the number of MCUs walked, or < 0.
extern "C" int phm_walk(const jsgpu_tables* tabs, const jsgpu_image_desc* desc, const uint8_t* scan, uint64_t n,
                        uint32_t* mcu_bit, int16_t* dc, uint32_t cap, uint32_t* ulen, uint32_t nseg_cap)
{
    Geo g;
    if (!make_geo(*desc, g)) return -1;
    static DevTableSet ts;
    build_table_set(*tabs, ts);
    std::vector<Interval> iv; std::vector<uint8_t> ub;
    unstuff(scan, n, g, iv, ub);
    uint32_t m = 0;
    for (uint32_t k = 0; k < g.nseg; k++) {
        Truth t;
        walk(ts, g, reinterpret_cast<const uint32_t*>(ub.data() + iv[k].uoff), iv[k].ulen, std::min(g.ri, g.nmcu - k * g.ri), t);
        if (k < nseg_cap) ulen[k] = iv[k].ulen;
        for (uint32_t i = 0; i < t.nmcu_done && m < cap; i++, m++) {
            mcu_bit[m] = t.mcu_bit[i]; dc[m * 3] = t.dc[i * 3]; dc[m * 3 + 1] = t.dc[i * 3 + 1]; dc[m * 3 + 2] = t.dc[i * 3 + 2];
        }
    }
    return (int)m;
}

// order: 0 = descending slot order (pure "previous round" reads), 1 = ascending, 2 = pseudo-random
// out[0] = mismatches, out[1] = fix rounds until settled, out[2] = slots in use, out[3] = virtual intervals,
// out[4] = slots whose guess was already right, out[5] = MCUs covered.  What the settled exit states reach (a slot's exit
// state is where its decoder stops: the first symbol start at or after the slot's end):
// out[6] = slots with no MCU start, out[7] = exits inside an MCU (block != 0), out[8] = exits inside a block (zig-zag != 0),
// out[9] = exits past the slot's end, out[10] = the largest overshoot in bits, out[11] = exits whose next symbol is an EOB,
// out[12] = the most MCU starts in one slot, out[13] = bit mask of the exit block indices 0..31, out[14] = ... 32..63,
// out[15] = mask of exit zig-zag indices 0..31, out[16] = ... 32..63, out[17] = slots that settled only after PH_MAX_ROUNDS
// fix rounds (their exit state last changed in a later round), out[18] = fix rounds that changed a slot after PH_MAX_ROUNDS
extern "C" int phm_check(const jsgpu_tables* tabs, const jsgpu_image_desc* desc, const uint8_t* scan, uint64_t n, int order, uint32_t* out)
{
    Geo g;
    if (!make_geo(*desc, g)) return -1;
    static DevTableSet ts;                                      // large
    build_table_set(*tabs, ts);
    std::vector<Interval> iv; std::vector<uint8_t> ub;
    unstuff(scan, n, g, iv, ub);
    // staged tables as the lane kernel lays them out
    uint32_t lslot[6], li[6], nl = 0;
    for (uint32_t c = 0; c < g.ns; c++) for (uint32_t cls = 0; cls < 2; cls++) {
        const uint32_t slot = cls ? g.sac[c] : g.sdc[c];
        uint32_t j = 0; while (j < nl && lslot[j] != slot) j++;
        if (j == nl) lslot[nl++] = slot;
        li[c * 2 + cls] = j;
    }
    std::vector<uint16_t> lutb((size_t)nl * JS_LANE_TAB, 0);
    for (uint32_t j = 0; j < nl; j++) {
        if (ts.lut2_overflow[lslot[j]] || ts.lut2_used[lslot[j]] > JS_LANE_L2S) return -2;      // the GPU path refuses such tables too
        memcpy(&lutb[(size_t)j * JS_LANE_TAB], ts.lut[lslot[j]], JS_LUT_SIZE * 2);
        memcpy(&lutb[(size_t)j * JS_LANE_TAB + JS_LUT_SIZE], ts.lut2[lslot[j]], ts.lut2_used[lslot[j]] * 2);
    }
    uint32_t qz[3][80]; uint16_t bdc[PH_MAX_BPM], bac[PH_MAX_BPM]; uint8_t bc[PH_MAX_BPM];
    uint32_t bi = 0;
    for (uint32_t c = 0; c < g.ns; c++) {
        for (uint32_t i = 0; i < 80; i++) qz[c][i] = (i < 64) ? ts.qz[g.dqt[c]][i] : ((64u + (i & 7)) << 16);
        for (uint32_t q = 0; q < g.H[c] * g.V[c] && bi < PH_MAX_BPM; q++, bi++) { bdc[bi] = (uint16_t)(li[c * 2] * JS_LANE_TAB); bac[bi] = (uint16_t)(li[c * 2 + 1] * JS_LANE_TAB); bc[bi] = (uint8_t)c; }
    }
    PhTabs t; t.lutb = lutb.data(); t.qz = &qz[0][0]; t.blk_dc = bdc; t.blk_ac = bac; t.blk_c = bc; t.bpm = bi; t.pshift = g.pshift;
    // slot arrays
    const uint64_t uregion = (n + (uint64_t)JS_USLACK * g.nseg + 128 + 255) / 256 * 256;
    const uint32_t nslots = (uint32_t)(uregion >> 9) + g.nseg + 2;
    std::vector<unsigned long long> x(nslots + 1, PH_DEAD); std::vector<uint32_t> ver(nslots + 1, 0), kk(nslots + 1, PH_NONE);
    std::vector<uint4> cnt(nslots + 1, make_uint4(0, 0, 0, 0)), aux(nslots + 1, make_uint4(0, 0, 0, 0)), pre(nslots + 1, make_uint4(0, 0, 0, 0));
    std::vector<uint32_t> st(g.nseg), ul(g.nseg); std::vector<unsigned long long> uo(g.nseg);
    for (uint32_t k = 0; k < g.nseg; k++) { st[k] = iv[k].s0; ul[k] = iv[k].ulen; uo[k] = iv[k].uoff; }
    PhSegs sg; sg.start = st.data(); sg.ulen = ul.data(); sg.uoff = uo.data(); sg.nseg = g.nseg;
    PhSlots a; a.x = x.data(); a.ver = ver.data(); a.k = kk.data(); a.cnt = cnt.data(); a.aux = aux.data(); a.pre = pre.data();
    std::vector<uint32_t> ord(nslots);
    for (uint32_t i = 0; i < nslots; i++) ord[i] = (order == 0) ? nslots - 1 - i : i;
    if (order == 2) { uint32_t r = 12345; for (uint32_t i = nslots; i > 1; i--) { r = r * 1664525u + 1013904223u; std::swap(ord[i - 1], ord[(r >> 8) % i]); } }
    for (uint32_t i = 0; i < nslots; i++) ph_guess_slot(t, sg, ub.data(), a, ord[i]);
    const std::vector<unsigned long long> xguess = x;
    uint32_t rounds = 0, late_rounds = 0;
    for (uint32_t r = 1; r < 100000; r++) {
        uint32_t nchg = 0;
        for (uint32_t i = 0; i < nslots; i++) nchg += ph_fix_slot(t, sg, ub.data(), a, ord[i], r) ? 1 : 0;
        rounds = r;
        if (r > PH_MAX_ROUNDS && nchg) late_rounds++;
        if (!nchg) break;
    }
    uint4 run = make_uint4(0, 0, 0, 0);                       // k_ph_scan
    for (uint32_t s = 0; s <= nslots; s++) {
        pre[s] = run;
        if (s < nslots) { run.x += cnt[s].x; run.y += cnt[s].y; run.z += cnt[s].z; run.w += cnt[s].w; }
    }
    // ---- check against the sequential walk ------------------------------------------------------------------------
    uint32_t bad = 0, used = 0, nv = 0, guessed = 0, covered = 0;
    std::vector<Truth> truth(g.nseg);
    std::vector<uint32_t> next_m(g.nseg);
    for (uint32_t k = 0; k < g.nseg; k++) {
        const uint32_t cntk = std::min(g.ri, g.nmcu - k * g.ri);
        walk(ts, g, reinterpret_cast<const uint32_t*>(ub.data() + iv[k].uoff), iv[k].ulen, cntk, truth[k]);
        next_m[k] = k * g.ri;
    }
    for (uint32_t s = 0; s < nslots; s++) {
        if (kk[s] == PH_NONE) continue;
        used++;
        if (x[s] == xguess[s]) guessed++;
        PhVseg v;
        if (!ph_vseg(sg, g.ri, g.nmcu, a, s, v)) continue;
        nv++;
        const Truth& T = truth[v.k];
        const uint32_t ml = v.m0 - v.k * g.ri;
        if (v.m0 != next_m[v.k]) { bad++; if (bad < 5) fprintf(stderr, "slot %u: starts at MCU %u, expected %u\n", s, v.m0, next_m[v.k]); }
        next_m[v.k] = v.m0 + v.nm;
        if (ml >= T.nmcu_done) { bad++; if (bad < 5) fprintf(stderr, "slot %u: MCU %u beyond the %u the walk found\n", s, ml, T.nmcu_done); continue; }
        if (v.bit != T.mcu_bit[ml]) { bad++; if (bad < 5) fprintf(stderr, "slot %u: MCU %u at bit %u, walk says %u\n", s, v.m0, v.bit, T.mcu_bit[ml]); }
        if ((int16_t)v.dc0 != T.dc[ml * 3] || (g.ns == 3 && ((int16_t)v.dc1 != T.dc[ml * 3 + 1] || (int16_t)v.dc2 != T.dc[ml * 3 + 2]))) {
            bad++; if (bad < 5) fprintf(stderr, "slot %u: DC predictors (%d,%d,%d), walk says (%d,%d,%d)\n", s, v.dc0, v.dc1, v.dc2, T.dc[ml * 3], T.dc[ml * 3 + 1], T.dc[ml * 3 + 2]);
        }
        covered += v.nm;
    }
    for (uint32_t k = 0; k < g.nseg; k++) {
        const uint32_t cntk = std::min(g.ri, g.nmcu - k * g.ri);
        if (iv[k].ulen && next_m[k] != k * g.ri + cntk) { bad++; if (bad < 5) fprintf(stderr, "interval %u: virtual intervals end at MCU %u, expected %u\n", k, next_m[k], k * g.ri + cntk); }
    }
    out[0] = bad; out[1] = rounds; out[2] = used; out[3] = nv; out[4] = guessed; out[5] = covered;
    // ---- what the settled exit states reach ---------------------------------------------------------------------------
    for (uint32_t i = 6; i < 19; i++) out[i] = 0;
    for (uint32_t s = 0; s < nslots; s++) {
        if (kk[s] == PH_NONE || x[s] == PH_DEAD) continue;
        const uint32_t k = kk[s], i = s - ph_slot_base(st[k], k), end = ul[k] * 8u;
        const uint32_t lim = std::min((i + 1) << PH_SUB_SHIFT, end);
        const uint32_t pos = ph_pos(x[s]), blk = ph_blk(x[s]), zz = ph_zz(x[s]);
        if (cnt[s].x == 0) out[6]++;
        out[12] = std::max(out[12], cnt[s].x);
        if (pos >= end) continue;                                   // the interval's end: no state inside the data
        if (blk) out[7]++;
        if (zz) out[8]++;
        if (pos > lim) { out[9]++; out[10] = std::max(out[10], pos - lim); }
        out[13 + (blk >> 5)] |= 1u << (blk & 31);
        out[15 + (zz >> 5)] |= 1u << (zz & 31);
        if (zz) {
            const uint32_t e = lookup(ts, g.sac[bc[blk]], peek(reinterpret_cast<const uint32_t*>(ub.data() + iv[k].uoff), pos));
            if (e && (e & 0xFF) == 0) out[11]++;
        }
        if (ver[s] > PH_MAX_ROUNDS) out[17]++;
    }
    out[18] = late_rounds;
    return 0;
}
