// wgmma.mma_async m64nNk16, fp16 x fp16 -> fp32, both operands K-major in shared memory (sm_90a), and the m64n32k16
// form with both operands MN-major (wgmma_tt_n32).
// One function per N the kernels use; the accumulator is the warpgroup's register fragment of a
// 64 x N tile: register i of thread (warp w, lane l) holds row 16 w + l / 4 + 8 ((i / 2) % 2),
// column 8 (i / 4) + 2 (l % 4) + i % 2.
#pragma once
#include <stdint.h>

namespace c2m {

template <int N> struct Wgmma;

template <> struct Wgmma<16> {
    // d: the first 8 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 8, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, "
            "%8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<32> {
    // d: the first 16 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 16, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "%16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<48> {
    // d: the first 24 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 24, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, "
            "%24, %25, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<64> {
    // d: the first 32 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 32, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "%32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<8> {
    // d: the first 4 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 4, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %6, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
            "{%0, %1, %2, %3}, "
            "%4, %5, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<24> {
    // d: the first 12 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 12, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %14, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n24k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, "
            "%12, %13, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<40> {
    // d: the first 20 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 20, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %22, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n40k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, "
            "%20, %21, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<56> {
    // d: the first 28 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 28, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %30, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n56k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27}, "
            "%28, %29, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<96> {
    // d: the first 48 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 48, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %50, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, "
            "%48, %49, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

template <> struct Wgmma<128> {
    // d: the first 64 registers of the accumulator (a longer array: its leading columns)
    template <int R>
    static __device__ __forceinline__ void mma(float (&d)[R], uint64_t da, uint64_t db, uint32_t accumulate) {
        static_assert(R >= 64, "accumulator too short");
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "%64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(accumulate)
            : "memory");
    }
};

// wgmma m64n32k16, fp16 x fp16 -> fp32, both operands MN-major in shared memory (imm-trans-a = imm-trans-b = 1);
// always accumulates (the caller zeroes the accumulator)
__device__ __forceinline__ void wgmma_tt_n32(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}

}  // namespace c2m
