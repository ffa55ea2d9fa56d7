// Wrappers of the wgmma shapes the kernels use (bf16 x bf16 -> fp32, m64 x N x 16).
//   wgmma_ss<N>     A and B from shared memory, both K-major (N = 16, 32, 64, 80, 96, 128, 144, 160, 176, 192, 256)
//   wgmma_rs_nN_tb  A from registers (the accumulator fragment of a previous product, packed to bf16), B MN-major
// d[] is the warpgroup's accumulator fragment: element i of thread (warp w, lane l) of the warpgroup holds row
// 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + i % 2.  acc = 0 overwrites d, else accumulates.
#pragma once
#include <stdint.h>

namespace sb200 {

template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t a, uint64_t b, uint32_t acc);

// Register lists of the generated shapes, in groups of eight fp32 registers: P<c> is the asm operand list of group c,
// D(c) its constraints; PL<n> / DL<n> the first n groups
#define SB200_WG_P0 "%0,%1,%2,%3,%4,%5,%6,%7"
#define SB200_WG_P1 ",%8,%9,%10,%11,%12,%13,%14,%15"
#define SB200_WG_P2 ",%16,%17,%18,%19,%20,%21,%22,%23"
#define SB200_WG_P3 ",%24,%25,%26,%27,%28,%29,%30,%31"
#define SB200_WG_P4 ",%32,%33,%34,%35,%36,%37,%38,%39"
#define SB200_WG_P5 ",%40,%41,%42,%43,%44,%45,%46,%47"
#define SB200_WG_P6 ",%48,%49,%50,%51,%52,%53,%54,%55"
#define SB200_WG_P7 ",%56,%57,%58,%59,%60,%61,%62,%63"
#define SB200_WG_P8 ",%64,%65,%66,%67,%68,%69,%70,%71"
#define SB200_WG_P9 ",%72,%73,%74,%75,%76,%77,%78,%79"
#define SB200_WG_P10 ",%80,%81,%82,%83,%84,%85,%86,%87"
#define SB200_WG_P11 ",%88,%89,%90,%91,%92,%93,%94,%95"
#define SB200_WG_P12 ",%96,%97,%98,%99,%100,%101,%102,%103"
#define SB200_WG_P13 ",%104,%105,%106,%107,%108,%109,%110,%111"
#define SB200_WG_P14 ",%112,%113,%114,%115,%116,%117,%118,%119"
#define SB200_WG_P15 ",%120,%121,%122,%123,%124,%125,%126,%127"
#define SB200_WG_D(c)                                                                                      \
  "+f"(d[8 * (c)]), "+f"(d[8 * (c) + 1]), "+f"(d[8 * (c) + 2]), "+f"(d[8 * (c) + 3]), "+f"(d[8 * (c) + 4]), \
      "+f"(d[8 * (c) + 5]), "+f"(d[8 * (c) + 6]), "+f"(d[8 * (c) + 7])
#define SB200_WG_PL1 SB200_WG_P0
#define SB200_WG_PL2 SB200_WG_PL1 SB200_WG_P1
#define SB200_WG_PL3 SB200_WG_PL2 SB200_WG_P2
#define SB200_WG_PL4 SB200_WG_PL3 SB200_WG_P3
#define SB200_WG_PL5 SB200_WG_PL4 SB200_WG_P4
#define SB200_WG_PL6 SB200_WG_PL5 SB200_WG_P5
#define SB200_WG_PL7 SB200_WG_PL6 SB200_WG_P6
#define SB200_WG_PL8 SB200_WG_PL7 SB200_WG_P7
#define SB200_WG_PL9 SB200_WG_PL8 SB200_WG_P8
#define SB200_WG_PL10 SB200_WG_PL9 SB200_WG_P9
#define SB200_WG_PL11 SB200_WG_PL10 SB200_WG_P10
#define SB200_WG_PL12 SB200_WG_PL11 SB200_WG_P11
#define SB200_WG_PL13 SB200_WG_PL12 SB200_WG_P12
#define SB200_WG_PL14 SB200_WG_PL13 SB200_WG_P13
#define SB200_WG_PL15 SB200_WG_PL14 SB200_WG_P14
#define SB200_WG_PL16 SB200_WG_PL15 SB200_WG_P15
#define SB200_WG_DL1 SB200_WG_D(0)
#define SB200_WG_DL2 SB200_WG_DL1, SB200_WG_D(1)
#define SB200_WG_DL3 SB200_WG_DL2, SB200_WG_D(2)
#define SB200_WG_DL4 SB200_WG_DL3, SB200_WG_D(3)
#define SB200_WG_DL5 SB200_WG_DL4, SB200_WG_D(4)
#define SB200_WG_DL6 SB200_WG_DL5, SB200_WG_D(5)
#define SB200_WG_DL7 SB200_WG_DL6, SB200_WG_D(6)
#define SB200_WG_DL8 SB200_WG_DL7, SB200_WG_D(7)
#define SB200_WG_DL9 SB200_WG_DL8, SB200_WG_D(8)
#define SB200_WG_DL10 SB200_WG_DL9, SB200_WG_D(9)
#define SB200_WG_DL11 SB200_WG_DL10, SB200_WG_D(10)
#define SB200_WG_DL12 SB200_WG_DL11, SB200_WG_D(11)
#define SB200_WG_DL13 SB200_WG_DL12, SB200_WG_D(12)
#define SB200_WG_DL14 SB200_WG_DL13, SB200_WG_D(13)
#define SB200_WG_DL15 SB200_WG_DL14, SB200_WG_D(14)
#define SB200_WG_DL16 SB200_WG_DL15, SB200_WG_D(15)

// wgmma_ss<N>: G = N / 16 register groups; the operands after them (a, b, acc) are numbered 8 G, 8 G + 1, 8 G + 2
#define SB200_WGMMA_SS(N, G, IA, IB, IACC)                                                                    \
  template <>                                                                                                 \
  __device__ __forceinline__ void wgmma_ss<N>(float* d, uint64_t a, uint64_t b, uint32_t acc) {               \
    static_assert(N == 16 * G && IA == 8 * G && IB == IA + 1 && IACC == IA + 2, "wgmma_ss register numbering"); \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #IACC ", 0;\n\t"                                   \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k16.f32.bf16.bf16 {" SB200_WG_PL##G "}, %" #IA ", %" #IB \
                 ", p, 1, 1, 0, 0;\n\t}\n"                                                                     \
                 : SB200_WG_DL##G                                                                             \
                 : "l"(a), "l"(b), "r"(acc));                                                                 \
  }
SB200_WGMMA_SS(16, 1, 8, 9, 10)
SB200_WGMMA_SS(32, 2, 16, 17, 18)
SB200_WGMMA_SS(64, 4, 32, 33, 34)
SB200_WGMMA_SS(80, 5, 40, 41, 42)
SB200_WGMMA_SS(96, 6, 48, 49, 50)
SB200_WGMMA_SS(128, 8, 64, 65, 66)
SB200_WGMMA_SS(144, 9, 72, 73, 74)
SB200_WGMMA_SS(160, 10, 80, 81, 82)
SB200_WGMMA_SS(176, 11, 88, 89, 90)
SB200_WGMMA_SS(192, 12, 96, 97, 98)
SB200_WGMMA_SS(256, 16, 128, 129, 130)
#undef SB200_WGMMA_SS

__device__ __forceinline__ void wgmma_rs_n64_tb(float* d, const uint32_t* a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}

}  // namespace sb200
