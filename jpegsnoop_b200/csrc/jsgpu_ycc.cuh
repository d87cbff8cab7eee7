// jsgpu_ycc.cuh — ConvertYCCtoRGBFastFloat (ImgDecode.cpp:4086-4139) on the device, written once for the fused tile kernel's
// exact path and colour tables, the simple kernels, the statistics and the channel preview.
#pragma once
#include <stdint.h>

// nValR = nValCr*(2-2*fConstRed)+nValY ... (:4289-4296 and :4118-4125), +128 included, one IEEE rounding per operation
// (the reference is built with -ffp-contract=off).  ConvertYCCtoRGB (jsgpu_preview.cu) shares it.
__device__ __forceinline__ void ycc_float_core(float y, float cb, float cr, float& vr, float& vg, float& vb)
{
    const float cR = 0.299f, cG = 0.587f, cB = 0.114f;
    const float kR = __fsub_rn(2.0f, __fmul_rn(2.0f, cR)), kB = __fsub_rn(2.0f, __fmul_rn(2.0f, cB));
    vr = __fadd_rn(__fmul_rn(cr, kR), y);
    vb = __fadd_rn(__fmul_rn(cb, kB), y);
    vg = __fdiv_rn(__fsub_rn(__fsub_rn(y, __fmul_rn(cB, vb)), __fmul_rn(cR, vr)), cG);
    vr = __fadd_rn(vr, 128.f); vb = __fadd_rn(vb, 128.f); vg = __fadd_rn(vg, 128.f);
}

// ConvertYCCtoRGBFastFloat of the samples py/pcb/pcr: y/cb/cr are the samples >> 3 clamped to -128..127 (nFinalY = y + 128),
// r/g/b the colour clamped to 0..255 and truncated.
struct YccFast { int y, cb, cr; uint32_t r, g, b; };
__device__ __forceinline__ YccFast ycc_fast(int py, int pcb, int pcr)
{
    YccFast o;
    o.y = max(-128, min(127, py >> 3)); o.cb = max(-128, min(127, pcb >> 3)); o.cr = max(-128, min(127, pcr >> 3));
    float vr, vg, vb; ycc_float_core((float)o.y, (float)o.cb, (float)o.cr, vr, vg, vb);
    o.r = (uint32_t)__float2int_rz(fminf(fmaxf(vr, 0.f), 255.f));
    o.g = (uint32_t)__float2int_rz(fminf(fmaxf(vg, 0.f), 255.f));
    o.b = (uint32_t)__float2int_rz(fminf(fmaxf(vb, 0.f), 255.f));
    return o;
}

// ... as a DIB word [B,G,R,0]
__device__ __forceinline__ uint32_t ycc_fast_bgra(int py, int pcb, int pcr)
{
    const YccFast o = ycc_fast(py, pcb, pcr);
    return o.b | (o.g << 8) | (o.r << 16);
}
