// jsgpu_phuff.cu — kernels of the self-synchronising Huffman passes for long restart intervals (scans without
// restart markers, BASELINE config 5; DRI of an MCU row or more).  The per-slot logic lives in
// jsgpu_phuff_core.cuh (shared with the host model of the CPU test-suite); this file stages the decode tables,
// maps threads to slots and enqueues the passes:
//
//   k_ph_sync<0>   guess: thread per 4096-bit slot, decode from the slot's first bit, store the exit state
//   k_ph_sync<1>   fix round r (PH_MAX_ROUNDS of them are enqueued; a round returns at once when the previous one
//                  changed nothing, and inside a round only slots whose predecessor changed decode again)
//   k_ph_fix_cta   safety net: if the last enqueued round still changed something, one CTA per image keeps
//                  iterating until its slots settle (never needed on well-formed data: a decoder locks onto the
//                  symbol grid within a few hundred bits, DESIGN.md §4)
//   k_ph_scan      per image: exclusive prefix sums of (MCU starts, DC sums) over its slots; clears the status
//                  words of its intervals
// Afterwards k_huff_lane<.., VSEG = true> (jsgpu_huff.cu) decodes every slot as a virtual restart interval.
// Reference semantics matched: CimgDecode::DecodeScanImg's serial MCU walk, ImgDecode.cpp:3164-3630.
#include "jsgpu_phuff_core.cuh"
#include <algorithm>

#define FULL 0xffffffffu
#define PH_THREADS 256

struct PhShared {
    LaneTabs t;
    uint32_t bpm, pshift;
    uint16_t blk_dc[PH_MAX_BPM], blk_ac[PH_MAX_BPM];
    uint8_t  blk_c[PH_MAX_BPM];
};
static_assert(sizeof(PhShared) % 16 == 0, "the staged tables behind PhShared are read as uint4");

// The image's MCU layout (thread 0, after lane_stage): which staged table every block of an MCU decodes with, its component,
// the blocks per MCU and the precision's divide.  It depends on the sampling factors and the precision, which (table_set,
// tab_sig) does not capture: images that share their staged tables can still differ here.
__device__ __forceinline__ void ph_layout(PhShared& sh, const DevImage& im)
{
    uint32_t bi = 0;
    for (uint32_t c = 0; c < im.ns; c++)
        for (uint32_t q = 0; q < im.H[c] * im.V[c] && bi < PH_MAX_BPM; q++, bi++) {
            sh.blk_dc[bi] = (uint16_t)(sh.t.li[c * 2] * JS_LANE_TAB); sh.blk_ac[bi] = (uint16_t)(sh.t.li[c * 2 + 1] * JS_LANE_TAB); sh.blk_c[bi] = (uint8_t)c;
        }
    sh.bpm = bi;
    sh.pshift = (im.precision > 8) ? im.precision - 8 : 0;
}

// Stage the image's decode tables and its MCU layout.
__device__ __forceinline__ void ph_stage(PhShared& sh, uint16_t* lutb, const DevImage& im, const DevTableSet* ts)
{
    __syncthreads();
    lane_stage(sh.t, lutb, im, ts);
    if (threadIdx.x == 0) ph_layout(sh, im);
    __syncthreads();
}

__device__ __forceinline__ PhTabs ph_tabs(const PhShared& sh, const uint16_t* lutb)
{
    PhTabs t; t.lutb = lutb; t.qz = &sh.t.qz[0][0]; t.blk_dc = sh.blk_dc; t.blk_ac = sh.blk_ac; t.blk_c = sh.blk_c; t.bpm = sh.bpm; t.pshift = sh.pshift;
    return t;
}
__device__ __forceinline__ PhSegs ph_segs(const DevBatch& b, const DevImage& im)
{
    PhSegs sg; sg.start = b.seg_start + im.seg_first; sg.ulen = b.seg_ulen + im.seg_first; sg.uoff = b.seg_uoff + im.seg_first; sg.nseg = im.nseg;
    return sg;
}
__device__ __forceinline__ PhSlots ph_slots(const DevBatch& b, const DevImage& im)
{
    PhSlots a; a.x = b.ph_x + im.ph_first; a.ver = b.ph_ver + im.ph_first; a.k = b.ph_k + im.ph_first;
    a.cnt = b.ph_cnt + im.ph_first; a.aux = b.ph_aux + im.ph_first; a.pre = b.ph_pre + im.ph_first;
    return a;
}

// MODE 0: guess.  MODE 1: fix round 1 (every slot).  MODE 2: fix round r >= 2 — only the slots whose predecessor changed in
// round r-1, taken from the per-image list that round wrote (dense threads instead of one live lane in a warp here and there).
template <int MODE>
__global__ void __launch_bounds__(PH_THREADS, 5) k_ph_sync(DevBatch b, uint32_t round)
{
    if (MODE == 2 && b.ph_nchg[round - 1] == 0) return;                    // the previous round changed nothing: settled
    extern __shared__ __align__(16) uint8_t ph_smem[];
    PhShared& sh = *reinterpret_cast<PhShared*>(ph_smem);
    uint16_t* const lutb = reinterpret_cast<uint16_t*>(ph_smem + sizeof(PhShared));
    uint32_t cur_sig = 0xffffffffu, cur_set = 0xffffffffu, cur_img = 0xffffffffu, nchg = 0;
    const uint32_t* const lin = b.ph_list[(round + 1) & 1]; const uint32_t* const nin = b.ph_nl[(round + 1) & 1];    // written by round - 1
    uint32_t* const lout = b.ph_list[round & 1]; uint32_t* const nout = b.ph_nl[round & 1];
    for (uint32_t it = blockIdx.x; it < b.nvitems; it += gridDim.x) {
        const uint2 item = b.vitems[it];                       // (image, first slot or first list position); PH_THREADS per item
        const DevImage& im = b.img[item.x];
        uint32_t nlist = 0;
        if (MODE == 2) { nlist = nin[item.x]; if (item.y >= nlist) continue; }     // CTA-uniform
        if (im.tab_sig != cur_sig || im.table_set != cur_set) {          // other decode tables: stage them and the layout
            ph_stage(sh, lutb, im, b.tables + im.table_set);
            cur_sig = im.tab_sig; cur_set = im.table_set; cur_img = item.x;
        } else if (item.x != cur_img) {                                    // same tables, another image: its own MCU layout
            __syncthreads();
            if (threadIdx.x == 0) ph_layout(sh, im);
            __syncthreads();
            cur_img = item.x;
        }
        uint32_t slot = item.y + threadIdx.x;
        if (MODE == 2) { if (slot >= nlist) continue; slot = lin[im.ph_first + slot]; }
        if (slot >= im.ph_nslots) continue;
        const PhTabs t = ph_tabs(sh, lutb);
        const PhSegs sg = ph_segs(b, im);
        const PhSlots a = ph_slots(b, im);
        if (MODE == 0) ph_guess_slot(t, sg, b.ubits, a, slot);
        else if (ph_fix_slot(t, sg, b.ubits, a, slot, round)) {
            nchg++;
            if (slot + 1 < im.ph_nslots && a.k[slot + 1] == a.k[slot]) lout[im.ph_first + atomicAdd(&nout[item.x], 1u)] = slot + 1;    // its successor decodes again next round
        }
    }
    if (MODE != 0) {
        nchg = __reduce_add_sync(FULL, nchg);
        if ((threadIdx.x & 31) == 0 && nchg) atomicAdd(&b.ph_nchg[round], nchg);
    }
}

__global__ void __launch_bounds__(PH_THREADS) k_ph_fix_cta(DevBatch b)
{
    if (b.ph_nchg[PH_MAX_ROUNDS] == 0) return;
    extern __shared__ __align__(16) uint8_t ph_smem[];
    PhShared& sh = *reinterpret_cast<PhShared*>(ph_smem);
    uint16_t* const lutb = reinterpret_cast<uint16_t*>(ph_smem + sizeof(PhShared));
    for (uint32_t ii = blockIdx.x; ii < b.nimg; ii += gridDim.x) {
        const DevImage& im = b.img[ii];
        if (!im.valid || !im.psync) continue;
        ph_stage(sh, lutb, im, b.tables + im.table_set);
        const PhTabs t = ph_tabs(sh, lutb);
        const PhSegs sg = ph_segs(b, im);
        const PhSlots a = ph_slots(b, im);
        for (uint32_t round = PH_MAX_ROUNDS + 1; ; round++) {
            int chg = 0;
            for (uint32_t slot = threadIdx.x; slot < im.ph_nslots; slot += blockDim.x) chg |= ph_fix_slot(t, sg, b.ubits, a, slot, round) ? 1 : 0;
            if (!__syncthreads_or(chg)) break;
        }
    }
}

// Per image: exclusive prefix sums of cnt over slots 0..ph_nslots (ph_nslots + 1 entries are written), and the status
// words of its intervals start at 0 (the lanes of k_huff_lane<VSEG> OR their findings in); an interval without data
// (a missing RSTn) is reported here because no slot stands for it.
__global__ void __launch_bounds__(256) k_ph_scan(DevBatch b)
{
    __shared__ uint4 s_w[8];
    __shared__ uint4 s_carry;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t ii = blockIdx.x; ii < b.nimg; ii += gridDim.x) {
        const DevImage& im = b.img[ii];
        if (!im.valid || !im.psync) continue;
        for (uint32_t k = threadIdx.x; k < im.nseg; k += blockDim.x) {
            const uint32_t gw = im.seg_first + k, ulen = b.seg_ulen[gw];
            b.seg_status[gw] = ulen ? 0u : 2u; b.seg_endbits[gw] = 0;
            if (!ulen) atomicOr(&b.img_status[ii], 2u);
        }
        const uint4* cnt = b.ph_cnt + im.ph_first; uint4* pre = b.ph_pre + im.ph_first;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = make_uint4(0, 0, 0, 0);
        __syncthreads();
        for (uint32_t base = 0; base <= im.ph_nslots; base += 256) {
            const uint32_t slot = base + threadIdx.x;
            const uint4 v = (slot < im.ph_nslots) ? cnt[slot] : make_uint4(0, 0, 0, 0);
            uint4 inc = v;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t x = __shfl_up_sync(FULL, inc.x, d), y = __shfl_up_sync(FULL, inc.y, d), z = __shfl_up_sync(FULL, inc.z, d), w = __shfl_up_sync(FULL, inc.w, d);
                if (lane >= (uint32_t)d) { inc.x += x; inc.y += y; inc.z += z; inc.w += w; }
            }
            if (lane == 31) s_w[wid] = inc;
            __syncthreads();
            uint4 wb = make_uint4(0, 0, 0, 0), tot = make_uint4(0, 0, 0, 0);
            #pragma unroll
            for (int q = 0; q < 8; q++) {
                const uint4 y = s_w[q];
                if (q < (int)wid) { wb.x += y.x; wb.y += y.y; wb.z += y.z; wb.w += y.w; }
                tot.x += y.x; tot.y += y.y; tot.z += y.z; tot.w += y.w;
            }
            const uint4 cy = s_carry;
            if (slot <= im.ph_nslots) pre[slot] = make_uint4(cy.x + wb.x + inc.x - v.x, cy.y + wb.y + inc.y - v.y, cy.z + wb.z + inc.z - v.z, cy.w + wb.w + inc.w - v.w);
            __syncthreads();
            if (threadIdx.x == 0) s_carry = make_uint4(cy.x + tot.x, cy.y + tot.y, cy.z + tot.z, cy.w + tot.w);
            __syncthreads();
        }
    }
}

int js_launch_selfsync(const DevBatch& b, int sm_count, cudaStream_t s)
{
    if (b.nvitems == 0) return 0;
    const size_t smem = sizeof(PhShared) + (size_t)b.lane_nlut * JS_LANE_TAB * 2;      // <= 20 KB: below the default dynamic limit
    const uint32_t grid = std::min<uint32_t>(b.nvitems, (uint32_t)sm_count * 8u);
    int n = 0;
    cudaMemsetAsync(b.ph_nchg, 0, (PH_MAX_ROUNDS + 2) * sizeof(uint32_t), s);
    cudaMemsetAsync(b.ph_nl[1], 0, (size_t)b.nimg * 4, s);
    k_ph_sync<0><<<grid, PH_THREADS, smem, s>>>(b, 0u); n++;
    k_ph_sync<1><<<grid, PH_THREADS, smem, s>>>(b, 1u); n++;
    for (uint32_t r = 2; r <= PH_MAX_ROUNDS; r++) {
        cudaMemsetAsync(b.ph_nl[r & 1], 0, (size_t)b.nimg * 4, s);
        k_ph_sync<2><<<grid, PH_THREADS, smem, s>>>(b, r); n++;
    }
    k_ph_fix_cta<<<std::min<uint32_t>(b.nimg, (uint32_t)sm_count * 4u), PH_THREADS, smem, s>>>(b); n++;
    k_ph_scan<<<std::min<uint32_t>(b.nimg, 65535u), 256, 0, s>>>(b); n++;
    return n;
}
