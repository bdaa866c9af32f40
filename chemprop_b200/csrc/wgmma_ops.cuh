// wgmma.mma_async wrappers (sm_90a), f32 accumulators in registers: d[i] of thread t of the warpgroup holds
// row 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) & 1), column 8 * (i / 4) + 2 * (t % 4) + (i & 1).
// One function per (shape, operand type, transpose) the kernels use; scale_d == 0 overwrites d instead of accumulating.
#pragma once
#include <stdint.h>

namespace dmpnn {
namespace tc {

// bf16 x bf16, both operands K-major
__device__ __forceinline__ void wgmma_bf16_n80(float (&d)[40], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39}, "
      "%40, %41, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_bf16_n152(float (&d)[76], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %78, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n152k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75}, "
      "%76, %77, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

// bf16 x bf16, both operands MN-major (transposed by the tensor core), d += a . b: one overload of wgmma_bf16_mn per width
// N = 16, 32, ..., 192, selected by the accumulator array's length N / 2.  The fragment of m64nNk16 is the n = 8 fragment
// repeated along N, so d[4 j + i] is the same element whatever N is.  An asm statement numbers its operands, so the
// register list and the constraint list grow by one 8-register piece per width; A, B, S name the three operands after them.
#define DMPNN_WG_D8(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define DMPNN_WG_R16 "%0,%1,%2,%3,%4,%5,%6,%7"
#define DMPNN_WG_R32 DMPNN_WG_R16 ",%8,%9,%10,%11,%12,%13,%14,%15"
#define DMPNN_WG_R48 DMPNN_WG_R32 ",%16,%17,%18,%19,%20,%21,%22,%23"
#define DMPNN_WG_R64 DMPNN_WG_R48 ",%24,%25,%26,%27,%28,%29,%30,%31"
#define DMPNN_WG_R80 DMPNN_WG_R64 ",%32,%33,%34,%35,%36,%37,%38,%39"
#define DMPNN_WG_R96 DMPNN_WG_R80 ",%40,%41,%42,%43,%44,%45,%46,%47"
#define DMPNN_WG_R112 DMPNN_WG_R96 ",%48,%49,%50,%51,%52,%53,%54,%55"
#define DMPNN_WG_R128 DMPNN_WG_R112 ",%56,%57,%58,%59,%60,%61,%62,%63"
#define DMPNN_WG_R144 DMPNN_WG_R128 ",%64,%65,%66,%67,%68,%69,%70,%71"
#define DMPNN_WG_R160 DMPNN_WG_R144 ",%72,%73,%74,%75,%76,%77,%78,%79"
#define DMPNN_WG_R176 DMPNN_WG_R160 ",%80,%81,%82,%83,%84,%85,%86,%87"
#define DMPNN_WG_R192 DMPNN_WG_R176 ",%88,%89,%90,%91,%92,%93,%94,%95"
#define DMPNN_WG_O16 DMPNN_WG_D8(0)
#define DMPNN_WG_O32 DMPNN_WG_O16, DMPNN_WG_D8(8)
#define DMPNN_WG_O48 DMPNN_WG_O32, DMPNN_WG_D8(16)
#define DMPNN_WG_O64 DMPNN_WG_O48, DMPNN_WG_D8(24)
#define DMPNN_WG_O80 DMPNN_WG_O64, DMPNN_WG_D8(32)
#define DMPNN_WG_O96 DMPNN_WG_O80, DMPNN_WG_D8(40)
#define DMPNN_WG_O112 DMPNN_WG_O96, DMPNN_WG_D8(48)
#define DMPNN_WG_O128 DMPNN_WG_O112, DMPNN_WG_D8(56)
#define DMPNN_WG_O144 DMPNN_WG_O128, DMPNN_WG_D8(64)
#define DMPNN_WG_O160 DMPNN_WG_O144, DMPNN_WG_D8(72)
#define DMPNN_WG_O176 DMPNN_WG_O160, DMPNN_WG_D8(80)
#define DMPNN_WG_O192 DMPNN_WG_O176, DMPNN_WG_D8(88)
#define DMPNN_WGMMA_BF16_MN(N, A, B, S)                                                                        \
  __device__ __forceinline__ void wgmma_bf16_mn(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc) {          \
    asm volatile(                                                                                              \
        "{\n\t.reg .pred p;\n\t"                                                                               \
        "setp.ne.b32 p, %" S ", 0;\n\t"                                                                        \
        "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 "                                            \
        "{" DMPNN_WG_R##N "}, %" A ", %" B ", p, 1, 1, 1, 1;\n\t}"                                             \
        : DMPNN_WG_O##N                                                                                        \
        : "l"(adesc), "l"(bdesc), "r"(1u));                                                                    \
  }
DMPNN_WGMMA_BF16_MN(16, "8", "9", "10")
DMPNN_WGMMA_BF16_MN(32, "16", "17", "18")
DMPNN_WGMMA_BF16_MN(48, "24", "25", "26")
DMPNN_WGMMA_BF16_MN(64, "32", "33", "34")
DMPNN_WGMMA_BF16_MN(80, "40", "41", "42")
DMPNN_WGMMA_BF16_MN(96, "48", "49", "50")
DMPNN_WGMMA_BF16_MN(112, "56", "57", "58")
DMPNN_WGMMA_BF16_MN(128, "64", "65", "66")
DMPNN_WGMMA_BF16_MN(144, "72", "73", "74")
DMPNN_WGMMA_BF16_MN(160, "80", "81", "82")
DMPNN_WGMMA_BF16_MN(176, "88", "89", "90")
DMPNN_WGMMA_BF16_MN(192, "96", "97", "98")
#undef DMPNN_WGMMA_BF16_MN

// tf32 x tf32 (K-major only)
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

}  // namespace tc
}  // namespace dmpnn
