// Hopper (sm_90a) tensor-core engine shared by the conv / weight-gradient / CLIP kernels: one 3xTF32 wgmma GEMM
// (or, with the compile-time operand mode PASSES = 1, its single-pass TF32 form, or with PASSES = TC_BF16 its bf16 form:
// see below)
//
//     D[m][n] = sum_k A[m][k] * B[n][k]        (fp32 operands, fp32-faithful result)
//
// whose operands and epilogue are supplied by an "op" (see the tc_*.cuh launchers), so that every contraction keeps its own
// addressing (tap shifts with per-sample zero padding, position-major weight-gradient operands, K slices) and its own fused
// epilogue without a copy of the pipeline.
//
// Three main loops share the wgmma wrappers, the tile layout and the numerics below: hc_conv_kernel (further down: TMA-fed,
// warp-specialised, persistent CTAs that walk the tiles) for the conv ops, whose A operand is a K-contiguous activation
// tile; hw_wgrad_kernel (the same pipeline,
// A transposed in registers, B transposed by the producer) for the conv weight gradient (WgradPOp); and hg_gemm_kernel
// (register-staged) for the other weight gradients and the CLIP GEMMs, whose M/N-contiguous operands are transposed on their
// way into shared memory.
//
// hg_gemm_kernel: one CTA = two warpgroups = one 128 x BN output tile (warpgroup g owns rows [64 g, 64 g + 64)); BN = 128,
// or 160 where the output width asks for it (hg_pick_bn).  Per K block of 32:
//   * every thread loads its share of the A and B tiles from global memory into registers one block AHEAD (the loads of
//     block kb+1 are in flight while the tensor cores work on block kb), splits each fp32 value x into tf32 pieces
//     hi = rna_tf32(x), lo = x - hi, and writes hi and lo into the 128-byte-swizzled K-major layout wgmma reads;
//     operands whose contiguous dimension is M/N (the position-major weight gradients) are transposed on that store;
//   * 4 x 3 wgmma.m64nBNk8.f32.tf32 per warpgroup: lo*hi + hi*lo + hi*hi (the lo*lo term is below fp32 resolution);
//   * the block's products are accumulated in a fresh register tile and then added into the running fp32 sum with
//     ordinary round-to-nearest FADDs.  The tensor core's internal accumulation truncates; chaining at most 12 MMAs per
//     block keeps that bias below 1e-7 relative however long K is, with no correction factor to calibrate per GPU.
//
// Both main loops take the pass count as a template argument: PASSES = 3 is the form above (the library's default, 1e-4
// parity with fp32), PASSES = 1 the TF32 form of the `_tf32` entry points (PyTorch's TF32 matmul precision): every fp32
// operand element is rounded once to tf32 (round to nearest, ties away from zero: the `hi` piece of the split), the stages
// hold no lo tiles, and ONE wgmma per k8 replaces the three.  The per-block fresh register tile and its round-to-nearest
// adds into the running sum are kept, so the accumulation bias bound and the fixed reduction order do not change.
// PASSES = TC_BF16 is the bf16 form of the `_bf16` entry points (torch.autocast with dtype bfloat16): every fp32 operand
// element is rounded once to bf16 (round to nearest even, cvt.rn.bf16x2.f32), the stages hold bf16 tiles of 64-byte rows
// with the 64-byte swizzle, and two wgmma.k16.bf16 per K block of 32 replace the tf32 MMAs.  Products of bf16 values are
// exact in fp32, and the per-block fresh tile and its round-to-nearest adds are kept here too.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <array>
#include <type_traits>
#include <utility>
#include <vector>
#include "common.cuh"

namespace bm {

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the attribute is per device, so a
// process-wide flag would leave a second device of the same process without it.  The table grows with the kernels a
// process launches: every instantiation of the tensor-core loops can reach it, so no fixed count bounds them.
inline int ensure_dyn_smem(const void* func, int bytes) {
    constexpr int kMaxDev = 64;
    static std::vector<std::pair<const void*, std::array<bool, kMaxDev>>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    size_t f = 0;
    while (f < done.size() && done[f].first != func) ++f;
    if (f == done.size()) done.push_back({func, {}});
    if (dev >= 0 && dev < kMaxDev && done[f].second[dev]) return 0;
    cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return set_error(3, "%s: cudaFuncSetAttribute: %s", __func__, cudaGetErrorString(e));
    if (dev >= 0 && dev < kMaxDev) done[f].second[dev] = true;
    return 0;
}


namespace tc {

// The operand modes of the main loops, carried by their template argument PASSES and the launchers' `passes`:
// TC_3XTF32 (three tf32 passes, the default forms), TC_TF32 (one tf32 pass, the `_tf32` forms) and TC_BF16 (one bf16
// pass, the `_bf16` forms)
constexpr int TC_3XTF32 = 3, TC_TF32 = 1, TC_BF16 = 2;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// fp32 -> (hi, lo) with hi = rna_tf32(x) and lo = rna_tf32(x - hi): x*y ~= hi*hi' + lo*hi' + hi*lo' to ~2^-21
__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// the same split with integer arithmetic: hi = x rounded to 10 mantissa bits (ties away), lo = x - hi exactly (the tensor
// core reads only lo's upper 19 bits: error <= 2^-21 |x|)
__device__ __forceinline__ void tf32_split(float x, float& hi, float& lo) {
    hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
    lo = x - hi;
}
// (lo, hi) -> two bf16 in one register, each rounded to nearest even, lo in the low half (the K order of a fragment)
__device__ __forceinline__ uint32_t bf16x2_rn(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
// four consecutive K elements as bf16, rounded to nearest even (8 bytes: x at the lowest address)
__device__ __forceinline__ uint2 bf16x4_rn(float4 v) { return make_uint2(bf16x2_rn(v.x, v.y), bf16x2_rn(v.z, v.w)); }

// ---------------------------------------------------------------------------------------------------
// wgmma
// ---------------------------------------------------------------------------------------------------
// K-major operand tile, rows of exactly 128 bytes (32 fp32), 128-byte swizzle, 8-row groups 1024 B apart (sm_90 layout)
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address
    d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;                    // stride byte offset: next 8-row group
    d |= (uint64_t)1 << 62;                              // SWIZZLE_128B
    return d;
}
// K-major bf16 operand tile, rows of exactly 64 bytes (32 bf16), 64-byte swizzle (16-byte chunk c of row r at chunk
// c ^ ((r >> 1) & 3)), 8-row groups 512 B apart; the tile starts 1 KB-aligned and a k16 step adds 32 bytes
__device__ __forceinline__ uint64_t wgmma_desc_k_sw64(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);        // start address
    d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(512 >> 4) << 32;                     // stride byte offset: next 8-row group
    d |= (uint64_t)2 << 62;                              // SWIZZLE_64B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// d (+)= A[smem] * B[smem]^T, M = 64, N = 128, K = 8, tf32 inputs, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32_m64n128(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
// the same with N = 160
__device__ __forceinline__ void wgmma_tf32_m64n160(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %82, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
        "%80, %81, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
          "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
          "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    static_assert(BN == 128 || BN == 160, "engine tile widths: 128, 160");
    if constexpr (BN == 128) wgmma_tf32_m64n128(d, adesc, bdesc, accumulate);
    else wgmma_tf32_m64n160(d, adesc, bdesc, accumulate);
}

// d (+)= A[registers] * B[smem]^T, M = 64, N = 128, K = 8: a = this thread's 4 tf32 values of the 64 x 8 A fragment
// (warp w of the group holds rows 16 w + lane/4 (+8 for a[1], a[3]), columns lane%4 (+4 for a[2], a[3]))
__device__ __forceinline__ void wgmma_tf32_rs_m64n128(float* d, const float* a, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
          "l"(bdesc), "r"(accumulate)
        : "memory");
}
// the same with N = 160
__device__ __forceinline__ void wgmma_tf32_rs_m64n160(float* d, const float* a, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %85, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
        "{%80, %81, %82, %83}, %84, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
          "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
          "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
          "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_tf32_rs(float* d, const float* a, uint64_t bdesc, int accumulate) {
    static_assert(BN == 128 || BN == 160, "engine tile widths: 128, 160");
    if constexpr (BN == 128) wgmma_tf32_rs_m64n128(d, a, bdesc, accumulate);
    else wgmma_tf32_rs_m64n160(d, a, bdesc, accumulate);
}

// The bf16 forms (TC_BF16): K = 16 per MMA, bf16 inputs, fp32 accumulators.  Shared-memory operands are K-major tiles of
// 64-byte rows (32 bf16: one K block) with the 64-byte swizzle (wgmma_desc_k_sw64); a register A fragment is 4 x 32 bits,
// each two bf16 of one row, the lower K index in the low half: register e of warp w holds row 16 w + lane/4 (+8 for e = 1,
// 3), K columns 2 (lane % 4) + {0, 1} (+8 for e = 2, 3).
__device__ __forceinline__ void wgmma_bf16_m64n128(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_bf16_m64n160(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %82, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
        "%80, %81, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
          "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
          "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_bf16_rs_m64n128(float* d, const uint32_t* a, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]),
          "l"(bdesc), "r"(accumulate)
        : "memory");
}

__device__ __forceinline__ void wgmma_bf16_rs_m64n160(float* d, const uint32_t* a, uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %85, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n160k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, "
        "{%80, %81, %82, %83}, %84, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),
          "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
          "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]),
          "l"(bdesc), "r"(accumulate)
        : "memory");
}
template <int BN>
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t adesc, uint64_t bdesc, int accumulate) {
    static_assert(BN == 128 || BN == 160, "engine tile widths: 128, 160");
    if constexpr (BN == 128) wgmma_bf16_m64n128(d, adesc, bdesc, accumulate);
    else wgmma_bf16_m64n160(d, adesc, bdesc, accumulate);
}
template <int BN>
__device__ __forceinline__ void wgmma_bf16_rs(float* d, const uint32_t* a, uint64_t bdesc, int accumulate) {
    static_assert(BN == 128 || BN == 160, "engine tile widths: 128, 160");
    if constexpr (BN == 128) wgmma_bf16_rs_m64n128(d, a, bdesc, accumulate);
    else wgmma_bf16_rs_m64n160(d, a, bdesc, accumulate);
}

// ---------------------------------------------------------------------------------------------------
// mbarrier / TMA
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, int bytes) {
    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Waits for the phase of `parity` to complete; false after HC_TIMEOUT_NS.  A correct pipeline waits microseconds at most,
// so a timeout means a lost arrival: the kernel reports it and exits instead of hanging the GPU.
constexpr uint64_t HC_TIMEOUT_NS = 4000000000ull;
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return true;
    const uint64_t t0 = globaltimer_ns();
    while (!mbar_try_wait(bar, parity))
        if (globaltimer_ns() - t0 > HC_TIMEOUT_NS) return false;
    return true;
}
// box (c0, c1, c2) of a 3D tensor map into shared memory; completes `bytes` on the mbarrier (out-of-bounds elements: 0)
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
                 : "memory");
}
// the same for a 2D tensor map
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
                 : "memory");
}

// ---------------------------------------------------------------------------------------------------
// per-phase probe of the warp-specialised loops (profiles/conv_phase_probe.py)
// ---------------------------------------------------------------------------------------------------
// Compiled only with -DBM_HC_PHASES (the shipped library never is: every method below is then empty).  Thread 0 of each
// warpgroup sums the SM clocks (%clock) spent in each phase over its CTA and adds them to g_hc_phases[kernel][phase]
// (kernel 0: hc_conv_kernel, 1: hw_wgrad_kernel), which bm_hc_phases() reads back.  Consumer phases are summed over both
// consumer warpgroups.  Each translation unit that includes this header gets its own copy of the counters: both kernels
// and bm_hc_phases() live in tc_conv_api.cu.
enum HcPhase {
    HP_FULL_WAIT,      // consumer: waiting on the full barrier
    HP_SPLIT_ADD,      // consumer: A fragment split + stage release + acc += part
    HP_MMA,            // consumer: wgmma issue to drain (wait_group 0)
    HP_EPI_LOAD,       // consumer epilogue: its loads (bias, addend, mask) until they are issued
    HP_EPI_STORE,      // consumer epilogue: the math and the stores (hw_wgrad_kernel: its whole epilogue)
    HP_EPI_STATS,      // consumer epilogue: BatchNorm statistics and max |output| after the last store
    HP_C_BLOCKS,       // consumer: K blocks (count)
    HP_TILES,          // consumer: tiles (count)
    HP_EMPTY_WAIT,     // producer: waiting on the empty barrier
    HP_B_LOAD,         // producer: B loads issued (or, loaded ahead, needed) until they are in registers
                       // (hw_wgrad_kernel: the wait for the block's staged dY slot)
    HP_STORE,          // producer: TMA issue, B split / stores, fence, arrive (hw_wgrad_kernel: + the producer barrier)
    HP_FIRST_FULL,     // producer: CTA start to its first full-barrier arrival
    HP_P_BLOCKS,       // producer: K blocks (count)
    HP_CTAS,           // CTAs (count, by the producer)
    HP_N
};
// one float4 of a B operand as loaded (tc_conv.cuh ConvOp::b_load): raw fp32 in h, or two pieces in h and l
struct HcB { float4 h, l; };
#ifdef BM_HC_PHASES
__device__ unsigned long long g_hc_phases[2][HP_N];
struct HcProbe {
    uint32_t start, t, acc[HP_N];
    __device__ static uint32_t now() {
        uint32_t c;
        asm volatile("mov.u32 %0, %%clock;" : "=r"(c));
        return c;
    }
    __device__ explicit HcProbe(uint32_t t0) : start(t0), t(now()) {
#pragma unroll
        for (int i = 0; i < HP_N; ++i) acc[i] = 0;
    }
    __device__ void mark(int p) { const uint32_t n = now(); acc[p] += n - t; t = n; }    // clocks since the last mark
    __device__ void count(int p) { acc[p] += 1; }
    __device__ void first_full() { if (acc[HP_FIRST_FULL] == 0) acc[HP_FIRST_FULL] = now() - start; }
    __device__ void ready(const float4& v) { asm volatile("" ::"f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)); }
    __device__ void ready(const HcB& v) { ready(v.h); ready(v.l); }
    __device__ void flush(int kernel) const {
        if (threadIdx.x % 128 != 0) return;
#pragma unroll
        for (int i = 0; i < HP_N; ++i)
            if (acc[i]) atomicAdd(&g_hc_phases[kernel][i], (unsigned long long)acc[i]);
    }
};
#else
struct HcProbe {
    __device__ static uint32_t now() { return 0; }
    __device__ explicit HcProbe(uint32_t) {}
    __device__ void mark(int) {}
    __device__ void count(int) {}
    __device__ void first_full() {}
    __device__ void ready(const float4&) {}
    __device__ void ready(const HcB&) {}
    __device__ void flush(int) const {}
};
#endif

// ---------------------------------------------------------------------------------------------------
// the GEMM engine
// ---------------------------------------------------------------------------------------------------
constexpr int HG_BM = 128, HG_BN = 128, HG_BK = 32, HG_THREADS = 256;
constexpr int HG_TILE_BYTES = 128 * HG_BK * 4;                        // 16 KB: 128 rows x 32 fp32
// one K block of a K-major operand tile of `rows` rows in shared memory: 32 tf32 (128-byte rows) or, for TC_BF16, 32 bf16
// (64-byte rows)
template <int PASSES> constexpr int hg_tile_bytes(int rows) { return rows * HG_BK * (PASSES == TC_BF16 ? 2 : 4); }
// one stage: A hi | A lo (128 rows each) | B hi | B lo (BN rows each), the lo tiles only when PASSES = 3 (TC_BF16: A and
// B as bf16); double-buffered, 1 KB alignment slack
template <int BN, int PASSES> constexpr int hg_stage_bytes() {
    return (PASSES == 3 ? 2 : 1) * (hg_tile_bytes<PASSES>(HG_BM) + hg_tile_bytes<PASSES>(BN));
}
template <int BN, int PASSES> constexpr int hg_smem_bytes() { return 2 * hg_stage_bytes<BN, PASSES>() + 1024; }

// The tile width for an output of n columns: 160 where it pads no more columns than 128 (320 columns: 2 exact tiles instead
// of 3 with 64 padding columns), else 128.
inline int hg_pick_bn(long long n) {
    const long long p128 = (n + 127) / 128 * 128, p160 = (n + 159) / 160 * 160;
    return p160 <= p128 ? 160 : 128;
}

// Operand fetch, per tile of ROWS rows (128 for A, BN for B) and K block (ops implement a4 / b4 with the signature below):
//   K-contiguous operand (Op::A_KCONTIG / B_KCONTIG):  v4(cta, kb, row, q) = elements k = 4q .. 4q+3 of tile row `row`
//   M/N-contiguous operand:                            v4(cta, kb, k, q)   = tile rows 4q .. 4q+3 at reduction index k
// Out-of-range elements (padding, tails, other samples) are returned as zeros.  store<PASSES> writes the tf32 pieces of a
// float4 into the hi and lo tiles (PASSES = 3) or its rounded value into the hi tile alone (PASSES = 1: `lo` is not touched;
// TC_BF16: rounded to bf16 into the 64-byte-row layout of wgmma_desc_k_sw64, 8 bytes per float4 of a K-contiguous operand,
// 2 bytes per element of a transposed one).
template <bool KCONTIG, int ROWS>
struct HgSlot {
    static constexpr int N4 = ROWS / 32;       // float4 moved per thread per tile
    // the N4 float4 this thread moves per ROWS x 32 tile: (i, q) = (row, k quad) or (k, row quad)
    __device__ static void coords(int tid, int j, int& i, int& q) {
        const int idx = tid + HG_THREADS * j;
        if (KCONTIG) { i = idx >> 3; q = idx & 7; }
        else {                                   // lanes: 8 k x 4 row quads (64 B contiguous per k, 2-way bank conflicts)
            const int lane = idx & 31, w = idx >> 5;
            i = (w & 3) * 8 + (lane & 7);
            q = (w >> 2) * 4 + (lane >> 3);
        }
    }
    template <int PASSES>
    __device__ static void store(uint8_t* hi, uint8_t* lo, int i, int q, float4 v) {
        if constexpr (PASSES == TC_BF16) {
            if (KCONTIG) {                             // row i, K elements 4q .. 4q+3: chunk q / 2, half q & 1
                *reinterpret_cast<uint2*>(hi + i * 64 + (((q >> 1) ^ ((i >> 1) & 3)) << 4) + (q & 1) * 8) = bf16x4_rn(v);
            } else {                                   // rows 4q .. 4q+3, K element i
                const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int r = 4 * q + c;
                    *reinterpret_cast<__nv_bfloat16*>(hi + r * 64 + (((i >> 3) ^ ((r >> 1) & 3)) << 4) + (i & 7) * 2) =
                        __float2bfloat16_rn(e[c]);
                }
            }
        } else if (KCONTIG) {
            float4 h, l;
            tf32_split(v.x, h.x, l.x); tf32_split(v.y, h.y, l.y); tf32_split(v.z, h.z, l.z); tf32_split(v.w, h.w, l.w);
            const int off = i * 128 + ((q ^ (i & 7)) << 4);
            *reinterpret_cast<float4*>(hi + off) = h;
            if (PASSES == 3) *reinterpret_cast<float4*>(lo + off) = l;
        } else {
            const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int r = 4 * q + c;
                const int off = r * 128 + (((i >> 2) ^ (r & 7)) << 4) + (i & 3) * 4;
                float h, l;
                tf32_split(e[c], h, l);
                *reinterpret_cast<float*>(hi + off) = h;
                if (PASSES == 3) *reinterpret_cast<float*>(lo + off) = l;
            }
        }
    }
};

// Accumulator fragment of warpgroup g (m64nBN, BN / 2 elements per thread): element i of thread (warp w of the group,
// lane) is
//   row 64 g + 16 w + lane/4 + 8 ((i >> 1) & 1),  column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
__device__ __forceinline__ int hg_row(int i) {
    const int w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    return 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);
}
__device__ __forceinline__ int hg_col(int i) { return 8 * (i >> 2) + 2 * (threadIdx.x & 3) + (i & 1); }

template <class Op, int BN, int PASSES>
__global__ void __launch_bounds__(HG_THREADS, 1) hg_gemm_kernel(const __grid_constant__ Op op) {
    static_assert(PASSES == TC_3XTF32 || PASSES == TC_TF32 || PASSES == TC_BF16, "3xTF32, single-pass TF32 or bf16");
    constexpr int NACC = BN / 2, STAGE = hg_stage_bytes<BN, PASSES>(), B_TILE = hg_tile_bytes<PASSES>(BN);
    constexpr int A_TILE = hg_tile_bytes<PASSES>(HG_BM);
    constexpr int A_LO = A_TILE, B_HI = (PASSES == 3 ? 2 : 1) * A_TILE;                 // tile offsets in a stage
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base_u32 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base_u32 - smem_u32(smem_raw));
    const int tid = threadIdx.x, wg = tid >> 7;
    using SA = HgSlot<Op::A_KCONTIG, HG_BM>;
    using SB = HgSlot<Op::B_KCONTIG, BN>;

    const typename Op::Cta cta = op.template cta<BN>();
    const int nkb = op.kblocks(cta);
    float4 ra[SA::N4], rb[SB::N4];
    auto fetch = [&](int kb) {
#pragma unroll
        for (int j = 0; j < SA::N4; ++j) {
            int i, q;
            SA::coords(tid, j, i, q);
            ra[j] = op.a4(cta, kb, i, q);
        }
#pragma unroll
        for (int j = 0; j < SB::N4; ++j) {
            int i, q;
            SB::coords(tid, j, i, q);
            rb[j] = op.b4(cta, kb, i, q);
        }
    };
    auto stash = [&](int s) {
        uint8_t* st = smem + s * STAGE;
#pragma unroll
        for (int j = 0; j < SA::N4; ++j) {
            int i, q;
            SA::coords(tid, j, i, q);
            SA::template store<PASSES>(st, st + A_LO, i, q, ra[j]);
        }
#pragma unroll
        for (int j = 0; j < SB::N4; ++j) {
            int i, q;
            SB::coords(tid, j, i, q);
            SB::template store<PASSES>(st + B_HI, st + B_HI + B_TILE, i, q, rb[j]);
        }
    };

    float acc[NACC], part[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    if (nkb > 0) {
        fetch(0);
        stash(0);
        fence_proxy_async();
        __syncthreads();
    }
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb & 1;
        if (kb + 1 < nkb) fetch(kb + 1);
        const uint32_t st = base_u32 + s * STAGE;
        const uint32_t a_hi = st + wg * (A_TILE / 2), a_lo = a_hi + A_LO;
        const uint32_t b_hi = st + B_HI, b_lo = b_hi + B_TILE;
        wgmma_fence();
        if constexpr (PASSES == TC_BF16) {
#pragma unroll
            for (int kk = 0; kk < HG_BK / 16; ++kk)       // 16 bf16 = 32 bytes along K inside the 64-byte swizzle span
                wgmma_bf16<BN>(part, wgmma_desc_k_sw64(a_hi + kk * 32), wgmma_desc_k_sw64(b_hi + kk * 32), kk != 0);
        } else {
#pragma unroll
            for (int kk = 0; kk < HG_BK / 8; ++kk) {
                const uint32_t off = kk * 32;              // 8 tf32 = 32 bytes along K inside the swizzle span
                const uint64_t dah = wgmma_desc_k_sw128(a_hi + off), dbh = wgmma_desc_k_sw128(b_hi + off);
                if constexpr (PASSES == 3) {
                    const uint64_t dal = wgmma_desc_k_sw128(a_lo + off), dbl = wgmma_desc_k_sw128(b_lo + off);
                    wgmma_tf32<BN>(part, dal, dbh, kk != 0);
                    wgmma_tf32<BN>(part, dah, dbl, 1);
                    wgmma_tf32<BN>(part, dah, dbh, 1);
                } else {
                    wgmma_tf32<BN>(part, dah, dbh, kk != 0);
                }
            }
        }
        wgmma_commit();
        if (kb + 1 < nkb) stash(s ^ 1);                    // the other stage's MMAs completed in the previous iteration
        wgmma_wait_all();
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] += part[i];
        fence_proxy_async();
        __syncthreads();
    }
    op.template epilogue<BN>(cta, acc, 64 * wg);
}

template <int BN, int PASSES, class Op>
inline int hg_run(const Op& op, dim3 grid, cudaStream_t st, const char* who) {
    constexpr int SMEM = hg_smem_bytes<BN, PASSES>();
    if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(hg_gemm_kernel<Op, BN, PASSES>), SMEM)) return rc;
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return 0;
    if (grid.y > 65535 || grid.z > 65535) return set_error(2, "%s: grid too large%s", who);
    hg_gemm_kernel<Op, BN, PASSES><<<grid, HG_THREADS, SMEM, st>>>(op);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", who, cudaGetErrorString(e));
    return 0;
}
// passes: TC_3XTF32, TC_TF32 or TC_BF16
template <int BN, class Op>
inline int hg_launch(const Op& op, dim3 grid, int passes, cudaStream_t st, const char* who) {
    if (passes == TC_BF16) return hg_run<BN, TC_BF16>(op, grid, st, who);
    return passes == 1 ? hg_run<BN, 1>(op, grid, st, who) : hg_run<BN, 3>(op, grid, st, who);
}
// the same with the tile width of hg_pick_bn
template <class Op>
inline int hg_launch_bn(int bn, const Op& op, dim3 grid, int passes, cudaStream_t st, const char* who) {
    return bn == 160 ? hg_launch<160>(op, grid, passes, st, who) : hg_launch<128>(op, grid, passes, st, who);
}

// ---------------------------------------------------------------------------------------------------
// the conv engine: the same 3xTF32 GEMM, warp-specialised and fed by TMA
// ---------------------------------------------------------------------------------------------------
// For ops whose A operand is a K-contiguous activation tile [1 sample][128 times][32 channels] of x [B][T][Cin] (ConvOp
// and its variants).  One CTA = one producer warpgroup + two consumer warpgroups, HC_STAGES stages, each with a full and
// an empty mbarrier.  The kernel is persistent: min(tiles, SMs) CTAs, CTA i computing tiles i, i + gridDim.x, ... of the
// op's tile list (Op::cta(tile): column tile fastest, so that the CTAs running together read the same weights from L2).
// The stage index and the barrier phases run on across tiles (one ring position per CTA), so the producer fills the next
// tile's stages while the consumers run the current tile's epilogue, and a tile pays no barrier set-up or pipeline fill.
//   * producer: thread 0 loads the A tile with TMA (op.a_box: the tap shift is in the t coordinate, and TMA's zero fill
//     outside [0, T) is the conv's zero padding); all 128 threads fetch B through op.b_load into registers, split it into
//     tf32 hi/lo and store both into the stage (128-byte-swizzled K-major, as in hg_gemm_kernel).  B is loaded one K block
//     ahead: block g+1's loads are issued as soon as block g is stored, so their L2 latency overlaps the wait for the next
//     free stage (the pre-split format, two loads per float4, loads the first half of the tile ahead and the second half
//     in turn, within the producer's register budget);
//   * consumers: warpgroup g reads its 64 raw fp32 A rows from the stage, splits them in registers with tf32_split and
//     issues 4 x 3 wgmma with A from registers: lo*hi + hi*lo + hi*hi per k8 into a fresh `part` tile, which is added into
//     `acc` with round-to-nearest FADDs per K block -- the pieces, MMA order and per-block adds of hg_gemm_kernel.
// Shared-memory traffic per K block at BN = 160: A 16 KB written by TMA + 16 KB read, B hi/lo 40 KB written + 120 KB
// read by the wgmmas (the register-staged loop also wrote A hi/lo and read A twice per MMA).
// PASSES = 1 (single-pass TF32): the producer stores B's rounded value alone (the pre-split format reads only its hi
// piece), the consumers round A in registers with cvt.rna and issue one wgmma per k8; B traffic: 20 KB written + 40 KB read.
// TC_BF16 (the bf16 form): the stage keeps the raw fp32 A tile that TMA writes (TMA cannot round) and B as bf16 in 64-byte
// rows with the 64-byte swizzle (wgmma_desc_k_sw64: 32 bf16 = one K block per row, so the 32-wide blocks, the stage count
// and the ring are unchanged).  The producer rounds B to bf16 on its store (the pre-split format: hi + lo, rounded once),
// the consumers convert their fp32 A fragment to bf16x2 registers and issue one k16 wgmma per 16 K; B traffic: 10 KB
// written + 20 KB read per block at BN = 160.
constexpr int HC_THREADS = 384, HC_CONSUMERS = 256, HC_STAGES = 3;
constexpr int HC_PRODUCER_REGS = 104, HC_CONSUMER_REGS = 200;    // 104 * 128 + 200 * 256 = 168 * 384 registers
// __launch_bounds__(HC_THREADS, 1) compiles the kernels for 168 registers per thread (65 536 / 384, rounded down to a
// multiple of 8), so the CTA holds 168 * 384 registers, not 65 536.  setmaxnreg.inc waits until the pool can grant its
// count: a split above that total would never start the consumers.
static_assert(HC_PRODUCER_REGS * 128 + HC_CONSUMER_REGS * HC_CONSUMERS <= (65536 / HC_THREADS) / 8 * 8 * HC_THREADS,
              "the producer / consumer register split must fit in the registers the CTA is launched with");
constexpr int HC_ERR_FULL = 901, HC_ERR_EMPTY = 902;           // status codes of a timed-out consumer / producer wait
// one stage: A raw fp32 (128 rows) | B hi | B lo (BN rows each; no lo tile when PASSES = 1, B as bf16 when TC_BF16),
// every tile 1 KB-aligned for the swizzle
template <int BN, int PASSES> constexpr int hc_stage_bytes() {
    return HG_TILE_BYTES + (PASSES == 3 ? 2 : 1) * hg_tile_bytes<PASSES>(BN);
}
template <int BN, int PASSES> constexpr int hc_smem_bytes() { return HC_STAGES * hc_stage_bytes<BN, PASSES>() + 1024; }

// index of a consumer thread in [0, 256) and a barrier over the consumer warpgroups only (the producer does not take part)
__device__ __forceinline__ int hc_consumer_tid() { return threadIdx.x - (HC_THREADS - HC_CONSUMERS); }
__device__ __forceinline__ void hc_consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(HC_CONSUMERS) : "memory"); }

// The stage ring's barriers (full[s], empty[s]), initialised by thread 0 before a __syncthreads
struct HcBars {
    uint64_t b[2 * HC_STAGES];
    __device__ void init() {
        for (int s = 0; s < HC_STAGES; ++s) {
            mbar_init(smem_u32(&b[s]), 128);                             // the producer's 128 threads (+ the TMA bytes)
            mbar_init(smem_u32(&b[HC_STAGES + s]), HC_CONSUMERS / 32);   // one arrival per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __device__ uint32_t full(int s) const { return smem_u32(&b[s]); }
    __device__ uint32_t empty(int s) const { return smem_u32(&b[HC_STAGES + s]); }
};

// One K block of a consumer warpgroup (hc_conv_kernel, hw_wgrad_kernel), where the numerics live: the warpgroup's 64 x 32
// A fragment, read raw through a(kk, e) (fp32 element e of k8 step kk in the register layout of wgmma_tf32_rs), is split
// into tf32 hi/lo in registers (PASSES = 1: rounded once with cvt.rna) and multiplied with the stage's B tiles at b_hi
// (hi) and b_hi + BN x 32 x 4 (lo): lo*hi + hi*lo + hi*hi per k8 into a fresh `part` tile (PASSES = 1: one wgmma per k8);
// once the MMAs have drained, release() hands the stage back and `part` is added into `acc` with round-to-nearest FADDs.
// TC_BF16: a(kk, e) is read as a float2 instead -- the fp32 elements of fragment register e of k16 step kk in the layout of
// wgmma_bf16_rs (row r0 + 8 (e & 1), K columns 16 kk + 8 (e >> 1) + 2 tq + {0, 1}) -- rounded to bf16x2 with
// cvt.rn and multiplied with the bf16 B tile at b_hi, one wgmma per k16.
// The two warpgroups issue their blocks concurrently: their 2 x 12 MMAs then take ~1900 clocks per block at BN = 160, the
// tensor floor; issuing them one warpgroup after the other measured slower (DESIGN §4.2).
template <int BN, int PASSES, class LoadA, class Release>
__device__ __forceinline__ void hc_consume_block(float* acc, float* part, uint32_t b_hi, const LoadA& a,
                                                 const Release& release, HcProbe& pr) {
    constexpr int NACC = BN / 2, B_TILE = BN * HG_BK * 4;
    if constexpr (PASSES == TC_BF16) {
        uint32_t r[2][4];                           // [k16][fragment register]: two bf16 each
#pragma unroll
        for (int kk = 0; kk < HG_BK / 16; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 v = a(kk, e);
                r[kk][e] = bf16x2_rn(v.x, v.y);
            }
        pr.mark(HP_SPLIT_ADD);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < HG_BK / 16; ++kk) wgmma_bf16_rs<BN>(part, r[kk], wgmma_desc_k_sw64(b_hi + kk * 32), kk != 0);
    } else if constexpr (PASSES == 3) {
        float hi[4][4], lo[4][4];                   // [k8][fragment element]
#pragma unroll
        for (int kk = 0; kk < HG_BK / 8; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) tf32_split(a(kk, e), hi[kk][e], lo[kk][e]);
        pr.mark(HP_SPLIT_ADD);
        const uint32_t b_lo = b_hi + B_TILE;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < HG_BK / 8; ++kk) {
            const uint32_t off = kk * 32;
            const uint64_t dbh = wgmma_desc_k_sw128(b_hi + off), dbl = wgmma_desc_k_sw128(b_lo + off);
            wgmma_tf32_rs<BN>(part, lo[kk], dbh, kk != 0);
            wgmma_tf32_rs<BN>(part, hi[kk], dbl, 1);
            wgmma_tf32_rs<BN>(part, hi[kk], dbh, 1);
        }
    } else {
        float r[4][4];                              // the same fragment, rounded once
#pragma unroll
        for (int kk = 0; kk < HG_BK / 8; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) r[kk][e] = tf32_rna(a(kk, e));
        pr.mark(HP_SPLIT_ADD);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < HG_BK / 8; ++kk) wgmma_tf32_rs<BN>(part, r[kk], wgmma_desc_k_sw128(b_hi + kk * 32), kk != 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    pr.mark(HP_MMA);
    release();
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] += part[i];
    pr.mark(HP_SPLIT_ADD);
}

template <class Op, int BN, int PASSES>
__global__ void __launch_bounds__(HC_THREADS, 1) hc_conv_kernel(const __grid_constant__ Op op,
                                                               const __grid_constant__ CUtensorMap xmap, int tiles) {
    static_assert(PASSES == TC_3XTF32 || PASSES == TC_TF32 || PASSES == TC_BF16, "3xTF32, single-pass TF32 or bf16");
    const uint32_t t_start = HcProbe::now();        // the probe's CTA start (BM_HC_PHASES)
    constexpr int NACC = BN / 2, STAGE = hc_stage_bytes<BN, PASSES>(), B_TILE = hg_tile_bytes<PASSES>(BN);
    extern __shared__ uint8_t smem_raw[];
    __shared__ HcBars bars;
    const uint32_t base_u32 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base_u32 - smem_u32(smem_raw));
    const int tid = threadIdx.x, wg = tid >> 7;
    if (tid == 0) bars.init();
    __syncthreads();

    if (wg == 0) {
        // ---- producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HC_PRODUCER_REGS));
        HcProbe pr(t_start);
        constexpr int NB4 = BN * HG_BK / 4 / 128;                 // float4 of B per thread per stage
        // one loop per weight format, so that the loads of a tile are issued back to back; PART float4 per thread are
        // loaded one block ahead (the pre-split format, 2 loads per float4: half of them)
        auto produce = [&](auto fmt) -> bool {
            constexpr int FMT = decltype(fmt)::value, PART = FMT == Op::B_SPLIT ? NB4 / 2 : NB4;
            int tile = blockIdx.x, kb = 0;
            typename Op::Cta cta = op.template cta<BN>(tile);
            // this thread's B elements j of a K block, the same in every block of the tile: tile column row + 16 j, k quad q
            const int row = (tid & 127) >> 3, q = tid & 7;        // tid < 128
            int boff[NB4];
            uint32_t live;
            auto columns = [&] {
                live = 0;
#pragma unroll
                for (int j = 0; j < NB4; ++j) {
                    const int o = op.template b_col<BN>(cta, row + 16 * j, q);
                    boff[j] = o < 0 ? 0 : o;                      // a column past the end loads column 0 and stores zeros
                    live |= (o >= 0 ? 1u : 0u) << j;
                }
            };
            HcB r[PART];
            auto load = [&](int p, long long base) {
#pragma unroll
                for (int j = 0; j < PART; ++j) r[j] = op.template b_load<FMT>(base + boff[p + j]);
            };
            columns();
            load(0, op.b_base(cta, 0));
            // the ring position: the stage (bits 0-1), the round through the ring mod 2 (bit 2), past the first round (bit 3)
            for (uint32_t sp = 0;; sp = (sp & 3) == HC_STAGES - 1 ? ((sp & 4) ^ 4) | 8 : sp + 1) {
                const int s = sp & 3;
                if ((sp & 8) && !mbar_wait(bars.empty(s), ((sp >> 2) & 1) ^ 1)) return false;
                pr.mark(HP_EMPTY_WAIT);
                const uint32_t st = base_u32 + s * STAGE, full = bars.full(s);
                if (tid == 0) {
                    const int3 c = op.a_box(cta, kb);
                    mbar_expect_tx(full, HG_TILE_BYTES);
                    tma_load_3d(st, &xmap, c.x, c.y, c.z, full);
                }
                uint8_t* bh = smem + s * STAGE + HG_TILE_BYTES;
                const long long base = op.b_base(cta, kb);
#pragma unroll
                for (int p = 0; p < NB4; p += PART) {
                    if (p > 0) load(p, base);
#pragma unroll
                    for (int j = 0; j < PART; ++j) pr.ready(r[j]);
                    pr.mark(HP_B_LOAD);
#pragma unroll
                    for (int j = 0; j < PART; ++j) {
                        const float4 v = (live >> (p + j)) & 1 ? op.template b_value<FMT>(cta, r[j])
                                                                : make_float4(0.f, 0.f, 0.f, 0.f);
                        HgSlot<true, BN>::template store<PASSES>(bh, bh + B_TILE, row + 16 * (p + j), q, v);
                    }
                    pr.mark(HP_STORE);
                }
                fence_proxy_async();                               // the generic-proxy stores, before the wgmmas read them
                mbar_arrive(full);
                pr.first_full();
                pr.count(HP_P_BLOCKS);
                if (++kb == op.kblocks(cta)) {                     // the CTA's next tile
                    tile += gridDim.x;
                    if (tile >= tiles) break;
                    cta = op.template cta<BN>(tile);
                    kb = 0;
                    columns();
                }
                load(0, op.b_base(cta, kb));                       // the next block's loads, in flight during the wait
                pr.mark(HP_STORE);
            }
            pr.mark(HP_STORE);
            return true;
        };
        const int f = op.b_format();
        bool ok;
        if constexpr (PASSES == 1)                      // raw or the hi piece of the split (rounding it again changes nothing);
            ok = produce(std::integral_constant<int, Op::B_RAW>());     // the launcher refuses the fp16 pieces
        else if constexpr (PASSES == TC_BF16)          // raw, or hi + lo of the split rounded once (no fp16 pieces either)
            ok = f == Op::B_RAW ? produce(std::integral_constant<int, Op::B_RAW>())
                                : produce(std::integral_constant<int, Op::B_SPLIT>());
        else
            ok = f == Op::B_RAW     ? produce(std::integral_constant<int, Op::B_RAW>())
                 : f == Op::B_SPLIT ? produce(std::integral_constant<int, Op::B_SPLIT>())
                                    : produce(std::integral_constant<int, Op::B_F16>());
        if (!ok && op.err) atomicCAS(op.err, 0, HC_ERR_EMPTY);
        pr.count(HP_CTAS);
        pr.flush(0);
        return;
    }
    // ---- consumers
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HC_CONSUMER_REGS));
    HcProbe pr(t_start);
    const int cg = wg - 1, lane = tid & 31, grp = lane >> 2, tq = lane & 3;
    const int r0 = 64 * cg + 16 * ((tid >> 5) & 3) + grp;        // A rows r0 and r0 + 8 of the fragment; r0 & 7 = grp
    // Fragment element e of k8 step kk is row r0 + 8 (e & 1), 16-byte chunk c = 2 kk + (e >> 1), word tq: word
    // 32 row + 4 (c ^ grp) + tq of the swizzled tile, i.e. (w0 ^ 4 c) + 256 (e & 1) with w0 = 32 r0 + 4 grp + tq (bits 2-4
    // of w0 hold grp alone), one register for all 16 addresses.
    const int w0 = 32 * r0 + 4 * grp + tq;
    // TC_BF16: the float2 of register e of k16 step kk is at word (wb ^ 4 (4 kk + 2 (e >> 1))) + 256 (e & 1): the chunk
    // bit tq / 2 joins grp in bits 2-4, which the XOR with the even chunk offset leaves in place
    const int wb = 32 * r0 + 4 * ((tq >> 1) ^ grp) + 2 * (tq & 1);
    float acc[NACC], part[NACC];
    // The ring position, packed into one register (the consumers' registers are taken by acc, part and the A fragment):
    // the stage (bits 0-1), the round through the ring mod 2 = the parity of the stage's full-barrier phase (bit 2) and the
    // tile's K blocks left (bits 3-)
    uint32_t pos = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
        for (pos |= (uint32_t)op.kblocks(op.template cta<BN>(tile)) << 3; pos >> 3; pos -= 8) {
            const int s = pos & 3;
            if (!mbar_wait(bars.full(s), (pos >> 2) & 1)) {
                if (op.err) atomicCAS(op.err, 0, HC_ERR_FULL);
                return;
            }
            pr.mark(HP_FULL_WAIT);
            pr.count(HP_C_BLOCKS);
            const float* at = reinterpret_cast<const float*>(smem + s * STAGE);
            hc_consume_block<BN, PASSES>(
                acc, part, base_u32 + s * STAGE + HG_TILE_BYTES,
                [&](int kk, int e) {
                    if constexpr (PASSES == TC_BF16)        // 16-byte chunk 4 kk + 2 (e >> 1) + tq / 2, words 2 (tq & 1) + {0, 1}
                        return *reinterpret_cast<const float2*>(at + ((wb ^ (4 * (4 * kk + 2 * (e >> 1)))) + 256 * (e & 1)));
                    else
                        return at[(w0 ^ (4 * (2 * kk + (e >> 1)))) + 256 * (e & 1)];
                },
                [&] {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bars.empty(s));
                },
                pr);
            pos = s == HC_STAGES - 1 ? (pos & ~7u) | ((pos & 4) ^ 4) : pos + 1;
        }
        op.template epilogue<BN, PASSES>(op.template cta<BN>(tile), acc, 64 * cg, pr);
        pr.mark(HP_EPI_STATS);
        pr.count(HP_TILES);
    }
    pr.flush(0);
}

// A dense fp32 tensor x of `rank` dimensions (dims[0] contiguous, no padding between rows) as a tensor map with the box
// box[0 .. rank), 128-byte swizzle (box[0] = 32 fp32: one 128-byte row), zero fill out of bounds
inline int hc_x_map(CUtensorMap* m, const float* x, int rank, const long long* dims, const int* box, const char* who) {
    using Encode = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static Encode encode = []() -> Encode {          // the driver's encoder, without linking libcuda
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return nullptr;
        return reinterpret_cast<Encode>(fn);
    }();
    if (!encode) return set_error(3, "%s: cuTensorMapEncodeTiled is not available%s", who);
    if (reinterpret_cast<uintptr_t>(x) & 15) return set_error(2, "%s: x must be 16-byte aligned%s", who);
    if (rank < 1 || rank > 5) return set_error(2, "%s: tensor map rank out of range%s", who);
    cuuint64_t d[5], strides[4];
    cuuint32_t b[5], elem[5];
    for (int i = 0; i < rank; ++i) {
        d[i] = (cuuint64_t)dims[i];
        b[i] = (cuuint32_t)box[i];
        elem[i] = 1;
        if (i > 0) strides[i - 1] = (i == 1 ? 4 : strides[i - 2]) * d[i - 1];
    }
    const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(x), d, strides, b, elem,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(2, "%s: cuTensorMapEncodeTiled failed%s", who);
    return 0;
}

// `tiles` output tiles (Op::cta(tile), tile in [0, tiles)) on min(tiles, SMs) persistent CTAs
template <int BN, int PASSES, class Op>
inline int hc_launch(const Op& op, long long tiles, cudaStream_t st, const char* who) {
    constexpr int SMEM = hc_smem_bytes<BN, PASSES>();
    if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(hc_conv_kernel<Op, BN, PASSES>), SMEM)) return rc;
    if (tiles <= 0) return 0;
    if (tiles >= (1ll << 31)) return set_error(2, "%s: too many tiles%s", who);
    CUtensorMap xmap;                                   // x [B][T][Cin], box [1][128][32]
    const long long dims[3] = {op.Cin, op.T, op.B};
    const int box[3] = {HG_BK, HG_BM, 1};
    if (int rc = hc_x_map(&xmap, op.x, 3, dims, box, who)) return rc;
    const int grid = (int)std::min<long long>(tiles, num_sms());
    hc_conv_kernel<Op, BN, PASSES><<<grid, HC_THREADS, SMEM, st>>>(op, xmap, (int)tiles);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", who, cudaGetErrorString(e));
    return 0;
}
// the tile width of hg_pick_bn and the operand mode op.passes (TC_3XTF32, TC_TF32 or TC_BF16; the fp16-piece weights
// only with TC_3XTF32)
template <class Op>
inline int hc_launch_bn(int bn, const Op& op, long long tiles, cudaStream_t st, const char* who) {
    if (op.passes == 1) {
        if (!op.w) return set_error(2, "%s: the single-pass form takes fp32 weights%s", who);
        return bn == 160 ? hc_launch<160, 1>(op, tiles, st, who) : hc_launch<128, 1>(op, tiles, st, who);
    }
    if (op.passes == TC_BF16) {
        if (!op.w) return set_error(2, "%s: the bf16 form takes fp32 weights%s", who);
        return bn == 160 ? hc_launch<160, TC_BF16>(op, tiles, st, who) : hc_launch<128, TC_BF16>(op, tiles, st, who);
    }
    return bn == 160 ? hc_launch<160, 3>(op, tiles, st, who) : hc_launch<128, 3>(op, tiles, st, who);
}

// ---------------------------------------------------------------------------------------------------
// the weight-gradient engine: the same GEMM, warp-specialised, for operands that are contiguous along M and N
// ---------------------------------------------------------------------------------------------------
// For WgradPOp (tc_wgradp.cuh): G[(tap, n)][m] = sum_p X[p + shift(tap), n] * dY[p, m] over flattened rows p = b T + t, with
// X [R][Nx] and dY [R][Mdy] channel-contiguous, while tf32 wgmma reads K-major shared-memory operands only.  The CTA shape,
// the stage layout (A raw | B hi | B lo), the full/empty mbarriers and the consumer block are hc_conv_kernel's:
//   * producer: thread 0 loads the A tile with TMA as 4 boxes [32 rows p][32 channels] of a 2D map over X (128-byte
//     swizzle).  Box j holds tile rows 32 j .. 32 j + 31, which are channels of ONE tap (Nx % 32 == 0), and is loaded at
//     row p0 + shift(tap); rows outside [0, R) arrive as zeros.  Thread 0 also loads block g+1's dY tile [32 p][BN m], as
//     BN / 32 boxes [32 p][32 m] of a 2D map over dY (128-byte swizzle; rows p >= R and columns m >= Mdy as zeros), into
//     a raw staging ring of 2 slots, apart from the stages, each slot with its own mbarrier.  All 128 threads then
//     transpose block g's slot into the K-major B tiles with 128-bit accesses (hw_transpose_dy) and store its tf32
//     pieces; a named barrier over the producer closes the block, so that every read of a slot precedes the TMA that
//     refills it;
//   * consumers read their A fragment transposed out of the boxes, zero the elements whose t + shift leaves [0, T) (sample
//     edges inside the flattened rows, which TMA cannot see) or whose p >= R, and run hc_consume_block.
// t = p mod T is carried from block to block (T >= 32: at most one sample edge per block), so the loop divides nothing.
// Op provides: R, T, X, Nx, dY, Mdy, err; cta<BN>(), kblocks(c), row0(c) (first flattened row of the CTA's K slice),
// a_box(c, j) = {first channel, tap shift} of box j (shift >= T for rows past the last tap), b_box(c, kb, j) = {first
// channel, first row} of dY box j of block kb, and epilogue<BN>(c, acc, m0).
// Shared memory per K block at BN = 160: A 16 KB written by TMA + 16 KB read; dY 20 KB written by TMA + 20 KB read by the
// producer; B 40 KB written + 120 KB read by the wgmmas.  HC_STAGES = 3 stages of 56 KB + 2 staging slots of 20 KB
// (209 KB per CTA at BN = 160, 3xTF32: a 4th stage no longer fits in 227 KB; the producer finishes a block in fewer
// clocks than the consumers and waits for free stages, so a deeper ring would not feed them faster).

// The producer's dY transpose, one K block: raw slot [BN / 32 boxes][32 p][32 m] (TMA's 128-byte swizzle: element (p, m)
// of a box at byte 128 p + 16 ((m / 4) ^ (p & 7)) + 4 (m & 3)) -> B tile [BN rows m][32 k = p] (K-major, the same swizzle:
// byte 128 m + 16 ((p / 4) ^ (m & 7)) + 4 (p & 3)).  The unit is a sub-block of 4 p x 4 m (p quad a, m quad c of a box):
// 4 LDS.128 of 4 m each, a register transpose, and per m one STS.128 of 4 p into B hi (and one into B lo), so every element
// keeps the position and the tf32 pieces of the scalar path.  A box has 64 sub-blocks, indexed by 6 bits s0 .. s5, with
//     c = s0 + 2 s2 + 4 s4,   a = s1 + 2 (s2 ^ s3) + 4 s5,
// and thread t takes sub-blocks t + 128 j.  A 128-bit access is served per quarter warp (8 lanes), which is conflict-free
// when its 8 lanes hit 8 distinct 16-byte bank groups: with 128-byte rows, the chunk index inside the row.  The 8 lanes of
// a quarter warp differ in s0, s1, s2 alone (s3, s4, s5 are lane bits 3, 4 and bit 5 of t):
//   * LDS of row p = 4 a + i (i = 0 .. 3): chunk c ^ (p & 7) = c ^ 4 s1 ^ i, bits (s0 ^ i0, s2 ^ i1, s4 ^ s1): 8 distinct;
//   * STS of row m = 4 c + e (e = 0 .. 3): chunk a ^ (m & 7) = a ^ 4 s0 ^ e, bits (s1 ^ e0, s2 ^ s3 ^ e1, s5 ^ s0): 8
//     distinct.
// (Plain c = s0 + 2 s1 + 4 s2 would leave the stores 4-way conflicted, since m & 7 sees only c's low bit; s2 feeding both
// c and a is what spreads both sides.)
// TC_BF16: the same sub-blocks and loads; per m one 8-byte store of the 4 p rounded to bf16, into the 64-byte-row B tile of
// wgmma_desc_k_sw64 (byte 64 m + 16 ((p / 8) ^ ((m / 2) & 3)) + 2 (p & 7)).
template <int BN, int PASSES>
struct HwTranspose {
    static constexpr int NSUB = 2 * BN, NJ = (NSUB + 127) / 128;     // sub-blocks per block, per thread (the last partly)
    int ro[NJ], bo[NJ];                                                // byte offsets in the raw slot and the B tile
    __device__ explicit HwTranspose(int t) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int idx = t + 128 * j, box = idx >> 6, s = idx & 63;
            const int c = (s & 1) | ((s >> 1) & 2) | ((s >> 2) & 4);
            const int a = ((s >> 1) & 1) | (((s >> 1) ^ (s >> 2)) & 2) | ((s >> 3) & 4);
            ro[j] = box * (32 * 128) + a * 512 + ((c ^ 4 * (a & 1)) << 4);     // row 4 a, chunk c ^ (4 a & 7)
            if constexpr (PASSES == TC_BF16)                                   // row 4 c, chunk (a / 2) ^ 2 (c & 1), half a & 1
                bo[j] = (32 * box + 4 * c) * 64 + (((a >> 1) ^ 2 * (c & 1)) << 4) + 8 * (a & 1);
            else
                bo[j] = (32 * box + 4 * c) * 128 + ((a ^ 4 * (c & 1)) << 4);  // row 4 c, chunk a ^ (4 c & 7)
        }
    }
    __device__ void run(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int t) const {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            if (NSUB % 128 != 0 && t + 128 * j >= NSUB) break;          // warp-uniform: the tail covers warps 0-1
            float v[4][4];                                             // [p][m] of the sub-block
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 r = *reinterpret_cast<const float4*>(raw + ((ro[j] + 128 * i) ^ (i << 4)));
                v[i][0] = r.x; v[i][1] = r.y; v[i][2] = r.z; v[i][3] = r.w;
            }
            if constexpr (PASSES == TC_BF16) {
#pragma unroll
                for (int e = 0; e < 4; ++e)                            // row 4 c + e: chunk bit 0 ^= e / 2
                    *reinterpret_cast<uint2*>(hi + ((bo[j] + 64 * e) ^ ((e >> 1) << 4))) =
                        bf16x4_rn(make_float4(v[0][e], v[1][e], v[2][e], v[3][e]));
                continue;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float4 h, l;
                tf32_split(v[0][e], h.x, l.x); tf32_split(v[1][e], h.y, l.y);
                tf32_split(v[2][e], h.z, l.z); tf32_split(v[3][e], h.w, l.w);
                const int off = (bo[j] + 128 * e) ^ (e << 4);
                *reinterpret_cast<float4*>(hi + off) = h;
                if (PASSES == 3) *reinterpret_cast<float4*>(lo + off) = l;
            }
        }
    }
};
// a barrier over the producer warpgroup's 128 threads only (id 2: hc_consumer_sync uses 1)
__device__ __forceinline__ void hw_producer_sync() { asm volatile("bar.sync 2, 128;" ::: "memory"); }
// the stages and 2 raw fp32 dY staging slots
template <int BN, int PASSES> constexpr int hw_smem_bytes() { return hc_smem_bytes<BN, PASSES>() + 2 * BN * HG_BK * 4; }

// bits a .. b-1 of a 32-bit mask (clamped to [0, 32))
__device__ __forceinline__ uint32_t hw_bits(int a, int b) {
    a = max(a, 0);
    b = min(b, 32);
    return a >= b ? 0u : (0xFFFFFFFFu >> (32 - (b - a))) << a;
}

template <class Op, int BN, int PASSES>
__global__ void __launch_bounds__(HC_THREADS, 1) hw_wgrad_kernel(const __grid_constant__ Op op,
                                                                const __grid_constant__ CUtensorMap xmap,
                                                                const __grid_constant__ CUtensorMap ymap) {
    static_assert(PASSES == TC_3XTF32 || PASSES == TC_TF32 || PASSES == TC_BF16, "3xTF32, single-pass TF32 or bf16");
    constexpr int NACC = BN / 2, STAGE = hc_stage_bytes<BN, PASSES>(), B_TILE = hg_tile_bytes<PASSES>(BN);
    const uint32_t t_start = HcProbe::now();        // the probe's CTA start (BM_HC_PHASES)
    constexpr int BOX_BYTES = HG_BK * HG_BK * 4;                 // one [32 p][32 channels] box of A or dY
    constexpr int RAW = HC_STAGES * STAGE, SLOT = BN * HG_BK * 4;   // the dY staging ring: 2 slots of raw fp32
    extern __shared__ uint8_t smem_raw[];
    __shared__ HcBars bars;
    __shared__ uint64_t dy_bars[2];                              // one per staging slot: thread 0's arrival + the TMA bytes
    const uint32_t base_u32 = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base_u32 - smem_u32(smem_raw));
    const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
    if (tid == 0) {
        mbar_init(smem_u32(&dy_bars[0]), 1);
        mbar_init(smem_u32(&dy_bars[1]), 1);
        bars.init();                                             // (its fence covers the two above)
    }
    __syncthreads();

    const typename Op::Cta cta = op.template cta<BN>();
    const int nkb = op.kblocks(cta), p0 = op.row0(cta), T = op.T;
    if (wg == 0) {
        // ---- producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(HC_PRODUCER_REGS));
        HcProbe pr(t_start);
        int bc[4], bs[4];                                // box j: channel and row shift (0 for a box of padding)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int2 b = op.a_box(cta, j);
            bc[j] = b.x;
            bs[j] = (b.y >= T || b.y <= -T) ? 0 : b.y;
        }
        const HwTranspose<BN, PASSES> tr(tid);
        auto stage_dy = [&](int kb) {                    // thread 0: block kb's dY boxes into staging slot kb & 1
            const uint32_t bar = smem_u32(&dy_bars[kb & 1]), slot = base_u32 + RAW + (kb & 1) * SLOT;
            mbar_expect_tx(bar, SLOT);
#pragma unroll
            for (int j = 0; j < BN / 32; ++j) {
                const int2 c = op.b_box(cta, kb, j);
                tma_load_2d(slot + j * BOX_BYTES, &ymap, c.x, c.y, bar);
            }
            mbar_arrive(bar);
        };
        if (tid == 0 && nkb > 0) stage_dy(0);
        for (int kb = 0; kb < nkb; ++kb) {
            const int s = kb % HC_STAGES, use = kb / HC_STAGES;
            // the next block's dY, in flight during this block's waits and transpose: its slot was last read by block
            // kb - 1, which the producer barrier closed
            if (tid == 0 && kb + 1 < nkb) stage_dy(kb + 1);
            if (use > 0 && !mbar_wait(bars.empty(s), (use - 1) & 1)) {
                if (op.err) atomicCAS(op.err, 0, HC_ERR_EMPTY);
                return;
            }
            pr.mark(HP_EMPTY_WAIT);
            const uint32_t st = base_u32 + s * STAGE, full = bars.full(s);
            if (tid == 0) {
                const int p = p0 + kb * HG_BK;
                mbar_expect_tx(full, HG_TILE_BYTES);
#pragma unroll
                for (int j = 0; j < 4; ++j) tma_load_2d(st + j * BOX_BYTES, &xmap, bc[j], p + bs[j], full);
            }
            pr.mark(HP_STORE);
            if (!mbar_wait(smem_u32(&dy_bars[kb & 1]), (kb >> 1) & 1)) {
                if (op.err) atomicCAS(op.err, 0, HC_ERR_EMPTY);
                return;
            }
            pr.mark(HP_B_LOAD);
            uint8_t* bh = smem + s * STAGE + HG_TILE_BYTES;
            tr.run(smem + RAW + (kb & 1) * SLOT, bh, bh + B_TILE, tid);
            fence_proxy_async();                               // the generic-proxy stores, before the wgmmas read them
            mbar_arrive(full);
            hw_producer_sync();                                // every read of this staging slot, before its next TMA
            pr.mark(HP_STORE);
            pr.first_full();
            pr.count(HP_P_BLOCKS);
        }
        pr.count(HP_CTAS);
        pr.flush(1);
        return;
    }
    // ---- consumers
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(HC_CONSUMER_REGS));
    HcProbe pr(t_start);
    const int cg = wg - 1, grp = lane >> 2, tq = lane & 3;
    const int r0 = 64 * cg + 16 * ((tid >> 5) & 3) + grp;        // A rows r0 and r0 + 8: one box, one tap
    const int sh = op.a_box(cta, r0 >> 5).y;
    const int tlo = max(0, -sh), thi = min(T, T - sh);          // t + shift in [0, T)  <=>  t in [tlo, thi)
    // word offset of fragment element e (row r0 + 8 (e & 1), k = tq + 4 (e >> 1)) at kk = 0; kk adds 8 rows of the box
    int off[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int c = (r0 & 31) + 8 * (e & 1), kq = tq + 4 * (e >> 1);
        off[e] = (r0 >> 5) * (BOX_BYTES / 4) + kq * 32 + (((c >> 2) ^ kq) << 2) + (c & 3);
    }
    // TC_BF16: word offset of the pair element i of fragment register e (row r0 + 8 (e & 1), k = 2 tq + i + 8 (e >> 1))
    // at kk = 0, indexed [e & 1][i]; e >> 1 adds 8 rows of the box and a k16 step kk 16
    int offb[2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int c = (r0 & 31) + 8 * h, kq = 2 * tq + i;
            offb[h][i] = (r0 >> 5) * (BOX_BYTES / 4) + kq * 32 + (((c >> 2) ^ kq) << 2) + (c & 3);
        }
    float acc[NACC], part[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    int t0 = p0 % T;                                            // t of the block's first row
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % HC_STAGES, use = kb / HC_STAGES;
        // rows k of this block that contribute: t0 + k in [tlo, thi), or in [tlo + T, thi + T) past the sample's end,
        // and p < R
        const int p = p0 + kb * HG_BK;
        const uint32_t live = ((hw_bits(tlo - t0, thi - t0) | hw_bits(tlo + T - t0, thi + T - t0)) & hw_bits(0, op.R - p)) >>
                              (PASSES == TC_BF16 ? 2 * tq : tq);
        t0 += HG_BK;
        if (t0 >= T) t0 -= T;
        if (!mbar_wait(bars.full(s), use & 1)) {
            if (op.err) atomicCAS(op.err, 0, HC_ERR_FULL);
            return;
        }
        pr.mark(HP_FULL_WAIT);
        pr.count(HP_C_BLOCKS);
        const float* at = reinterpret_cast<const float*>(smem + s * STAGE);
        hc_consume_block<BN, PASSES>(
            acc, part, base_u32 + s * STAGE + HG_TILE_BYTES,
            [&](int kk, int e) {
                if constexpr (PASSES == TC_BF16) {
                    const int d = 8 * 32 * (e >> 1) + 16 * 32 * kk, k = 16 * kk + 8 * (e >> 1);
                    const float v0 = at[offb[e & 1][0] + d], v1 = at[offb[e & 1][1] + d];
                    return make_float2((live >> k) & 1 ? v0 : 0.f, (live >> (k + 1)) & 1 ? v1 : 0.f);
                } else {
                    const float v = at[off[e] + 8 * 32 * kk];
                    return (live >> (8 * kk + 4 * (e >> 1))) & 1 ? v : 0.f;
                }
            },
            [&] {
                __syncwarp();
                if (lane == 0) mbar_arrive(bars.empty(s));
            },
            pr);
    }
    op.template epilogue<BN>(cta, acc, 64 * cg);
    pr.mark(HP_EPI_STORE);
    pr.count(HP_TILES);
    pr.flush(1);
}

template <int BN, int PASSES, class Op>
inline int hw_launch(const Op& op, dim3 grid, cudaStream_t st, const char* who) {
    constexpr int SMEM = hw_smem_bytes<BN, PASSES>();
    if (int rc = ensure_dyn_smem(reinterpret_cast<const void*>(hw_wgrad_kernel<Op, BN, PASSES>), SMEM)) return rc;
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return 0;
    if (grid.y > 65535 || grid.z > 65535) return set_error(2, "%s: grid too large%s", who);
    CUtensorMap xmap, ymap;                             // X [R][Nx] and dY [R][Mdy], boxes [32][32]
    const long long xdims[2] = {op.Nx, op.R}, ydims[2] = {op.Mdy, op.R};
    const int box[2] = {HG_BK, HG_BK};
    if (int rc = hc_x_map(&xmap, op.X, 2, xdims, box, who)) return rc;
    if (op.Mdy % 4 != 0) return set_error(2, "%s: dy rows must be a multiple of 16 bytes%s", who);
    if (int rc = hc_x_map(&ymap, op.dY, 2, ydims, box, who)) return rc;
    hw_wgrad_kernel<Op, BN, PASSES><<<grid, HC_THREADS, SMEM, st>>>(op, xmap, ymap);
    ++g_launches;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(3, "%s: launch failed: %s", who, cudaGetErrorString(e));
    return 0;
}
// tile width 160 or 128 (hg_pick_bn), passes TC_3XTF32, TC_TF32 or TC_BF16
template <class Op>
inline int hw_launch_bn(int bn, const Op& op, dim3 grid, int passes, cudaStream_t st, const char* who) {
    if (passes == TC_BF16)
        return bn == 160 ? hw_launch<160, TC_BF16>(op, grid, st, who) : hw_launch<128, TC_BF16>(op, grid, st, who);
    if (passes == 1) return bn == 160 ? hw_launch<160, 1>(op, grid, st, who) : hw_launch<128, 1>(op, grid, st, who);
    return bn == 160 ? hw_launch<160, 3>(op, grid, st, who) : hw_launch<128, 3>(op, grid, st, who);
}

// the plain epilogue: D[z plane][row][col] = acc for rows < rows, cols < cols (row-major, leading dimension ld)
struct HgStore {
    float* D;
    long long ld;
    int rows, cols;
    template <int BN>
    __device__ void store(const float* acc, int m0, int n0) const {
#pragma unroll
        for (int i = 0; i < BN / 2; i += 2) {
            const int r = m0 + hg_row(i), c = n0 + hg_col(i);
            if (r >= rows) continue;
            float* d = D + (long long)r * ld + c;
            if (c + 1 < cols && ((reinterpret_cast<uintptr_t>(d) & 7) == 0)) {
                *reinterpret_cast<float2*>(d) = make_float2(acc[i], acc[i + 1]);
            } else {
                if (c < cols) d[0] = acc[i];
                if (c + 1 < cols) d[1] = acc[i + 1];
            }
        }
    }
};

}  // namespace tc

}  // namespace bm
