// valuenet_tc.cuh — the reference value network (model/model_vv.py:13-52) on Hopper tensor cores (sm_90a, wgmma).
//
// Precision: north_star asks value outputs within 1e-5 of the reference's fp32.  Plain bf16/tf32/fp16 MMAs cannot
// reach that, so every fp32 operand x is split into two fp16 terms x = x1 + x2 (11 + 11 = 22 mantissa bits, the
// precision class of 3xTF32) and each product a*b is accumulated in fp32 as a1*b2 + a2*b1 + a1*b1 (the dropped
// a2*b2 is < 2^-22 relative).  Operands are pre-scaled by exact powers of two (activations x16, weights x64) so that the
// low terms stay in fp16's normal range; the epilogues undo the 2^10.  Three fp16 MMAs replace one fp32 product.
//
//   k_tc_conv  persistent CTAs of TCC_WGS warpgroups; each warpgroup carries its own boards through the whole stack:
//              obs key -> im2col (exact fp16) -> conv1 as one K=16 wgmma per 64-row tile -> epilogue (bias, ReLU, split) -> smem
//              conv2 / conv3 as shift-GEMMs: activations live in shared memory channel-chunk-major
//              ([8-channel chunk][pixel row][16 B]), so the A operand of a filter tap is the SAME array started a few rows
//              later — a no-swizzle K-major operand layout with SBO = 128 B, LBO = rows*16 B.  conv2 runs on an 8-wide
//              row-major grid with the three horizontal taps stacked along N (N = 96) and summed by two lane shuffles; conv3
//              runs on a column-major grid of column height 16, where its 56 outputs fit one 64-row tile (see below).
//              wgmma.mma_async (M=64 pixels, K=16) from shared-memory descriptors, accumulators in registers; the epilogues
//              apply bias+ReLU, re-split (fp16 x2) and write the next layer's operand (or act3 to HBM in the FC kernel's tile layout).
//   k_tc_fc    [R,1792] x [1792,256]: 128-row tiles, operands streamed by cp.async.bulk (1-D TMA) into an mbarrier ring —
//              both operands are stored in HBM already in the no-swizzle K-major layout, so one bulk copy per operand block needs
//              no tensor map; one producer warp, two consumer warpgroups (64 rows each, N = 256 accumulators in registers);
//              the epilogue fuses bias+ReLU+fc_out+sigmoid+affine and scatters (v, var) to the requesting tree slot.
//
// Both kernels take the number of fp16 terms per operand, NT, as a template argument.  NT = 2 is the split above (eval_kind net_tc).
// NT = 1 (eval_kind net_fp16) keeps only x1 of every activation and weight and issues the single product a1*b1: conv1 runs at N = 32
// (the second weight term is no longer stacked along N), conv2 / conv3 / fc1 issue one MMA where the split issues three, the epilogues
// round to one fp16, and act3 in HBM is one plane.  Same scaling, same layouts (the x2 slots stay allocated and are not read), so the
// overflow and subnormal limits of the split carry over; each rounded operand is exact to 2^-11 relative instead of 2^-22.
#pragma once
#include <cuda_fp16.h>
#include "gmma.cuh"
#include "search_dev.cuh"
#include "valuenet_simt.cuh"

namespace b200 {

constexpr float TC_SCALE_A = 16.f, TC_SCALE_W = 64.f, TC_UNSCALE = 1.f / 1024.f;

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, fp16 operands from shared memory (both K-major), fp32 accumulators: thread t of the
// warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8j + 2*(t%4) (+1) in d[4j + {0,1}] (row) / d[4j + {2,3}] (row + 8).
// accumulate == 0 overwrites D.
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
        "}, %16, %17, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n96(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
        "}, %48, %49, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
        "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
        "}, %128, %129, p, 1, 1, 0, 0;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// x = x1 + x2 with fp16 terms (round-to-nearest each step); two fp32 values -> one 32-bit word per split
__device__ __forceinline__ void split2(float x0, float x1, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 f = __half22float2(h);
    const __half2 l = __floats2half2_rn(x0 - f.x, x1 - f.y);
    hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
}
// the NT = 1 form: x ~= x1, one fp16 per value (round-to-nearest)
__device__ __forceinline__ uint32_t round1(float x0, float x1) {
    const __half2 h = __floats2half2_rn(x0, x1);
    return *reinterpret_cast<const uint32_t *>(&h);
}

// ---------------------------------------------------------------------------------------------------- conv kernel
// In conv2 the three horizontal taps (dx) of a 3x3 filter are stacked along N, so the layer is a few wide MMAs instead of many narrow ones:
//   D'[p][dx*32 + cout] = sum_{dy, cin} act[p + dy*8][cin] * W[dy][dx][cin][cout]          (A operand shifted by dy*8 rows only)
//   out[p][cout]        = D'[p][0*32+cout] + D'[p+1][1*32+cout] + D'[p+2][2*32+cout]        (epilogue: two lane shuffles)
// conv1 and conv2 live on an 8-wide pixel grid (p = y*8 + x).  In the wgmma accumulator layout pixel x of a row sits in lanes 4x..4x+3,
// so p+1 / p+2 are 4 / 8 lanes further in the same register, and p+dx never leaves the row.  conv2 is 18 MMAs per 64-row tile
// (3 dy x 2 channel halves x 3 split products, N = 96), two tiles; conv1 (K = 9 taps, exact {-1,0,1} inputs) runs on the tensor core
// too, from an im2col operand the warpgroup builds.
// conv3 has only 14x4 valid outputs, which the 8-wide grid spreads over two tiles.  Its input (act2) and output use a column-major grid
// of column height 16 instead (q = x*16 + y): every valid output has p <= 61, one 64-row tile, and tap (dy, dx) reads row p + 16 dx + dy.
// The three dx taps get an accumulator each (N = 32), so no shuffles are needed:
//   D_dx[p][cout] = sum_{dy, cin} act2[p + 16 dx + dy][cin] * W[dy][dx][cin][cout],    out[p] = (D_2 + D_1) + D_0
// Each D_dx receives exactly the MMA sequence (dy, half, split product) that the N = 96 form issued into its 32 columns, from the same
// operands, so act3 is the same bits as with two N = 96 tiles, for 54 n32 MMAs per board instead of 36 n96.
constexpr int TCC_WGS = 4;                  // warpgroups per CTA; each evaluates its own boards from key to act3
constexpr int TCC_THREADS = TCC_WGS * 128;
constexpr int TCC_R = 144;                  // act1 rows per board: the 18x8 grid of conv1's outputs
constexpr int TCC_WBLOCK = 2 * 2 * 96 * 16;  // conv2: one (dy, channel half) block: [weight split 2][chunk 2][n = dx*32 + cout][16 B]
constexpr int TCC_WBYTES = 6 * TCC_WBLOCK;   // one conv layer = 36864 B
constexpr int TCC_W3BLOCK = 2 * 32 * 16;     // conv3: one (dx, dy, channel half, weight split) block: [chunk 2][cout 32][16 B]
static_assert(36 * TCC_W3BLOCK == TCC_WBYTES, "conv3 weight layout");
constexpr int TCC_W1BYTES = 2 * 64 * 16;     // conv1: [chunk 2][n = split*32 + cout][16 B], k = tap (9 of 16 used)
constexpr int TCC_RUN = 4;                  // consecutive requests handed to a warpgroup at a time
constexpr int TCC_ASLOT = 2 * 4 * TCC_R * 16;    // act1 of one board: [split][chunk 4][144 rows][16 B]
// act2 of one board: [split][chunk 4][98 rows][16 B], row q = x*16 + y (x < 6, y < 16) plus rows 96..97, which conv3's dy shift reads
// for discarded outputs only (zeroed once).  98 = 2 (mod 8) puts the four chunks 8 banks apart, and the split stride of 4*98*16 + 16 B
// puts the second term 4 banks from the first: the eight words a lane stores per pixel fall on eight disjoint 4-bank groups.
constexpr int TCC_R2 = 98;
constexpr int TCC_A2SPLIT = 4 * TCC_R2 * 16 + 16;
constexpr int TCC_A2SLOT = 2 * TCC_A2SPLIT;
static_assert((TCC_R2 * 4) % 32 == 8 && (TCC_A2SPLIT / 4) % 32 == 4, "act2 bank layout");
constexpr int TCC_IMROWS = 192;             // im2col rows per board: 144 used, three 64-row tiles
constexpr int TCC_IMSLOT = 2 * TCC_IMROWS * 16;  // [chunk 2][192 rows][16 B] fp16
constexpr int TCC_OFF_W2 = 0;
constexpr int TCC_OFF_W3 = TCC_OFF_W2 + TCC_WBYTES;
constexpr int TCC_OFF_W1 = TCC_OFF_W3 + TCC_WBYTES;
constexpr int TCC_OFF_A1 = TCC_OFF_W1 + TCC_W1BYTES;
constexpr int TCC_OFF_IM = TCC_OFF_A1 + TCC_WGS * TCC_ASLOT;
constexpr int TCC_OFF_A2 = TCC_OFF_IM + TCC_WGS * TCC_IMSLOT;
constexpr int TCC_OFF_BIAS = TCC_OFF_A2 + TCC_WGS * TCC_A2SLOT;    // 96 floats, pre-scaled by TC_SCALE_A
constexpr int TCC_OFF_KEY = TCC_OFF_BIAS + 96 * 4;                  // TCC_WGS x 32 words: row table (20 rows: settled | piece << 16)
constexpr int TCC_SMEM = TCC_OFF_KEY + TCC_WGS * 32 * 4;
constexpr int ACT3_KCHUNKS = 224;           // 1792 / 8
static_assert(TCC_SMEM <= 227 * 1024, "k_tc_conv shared memory");

// MMA work issued per board, in n-units: one column of an m64 k16 wgmma = 64 * 16 * 2 = 2048 FLOP.  NT = 2 / NT = 1:
//   conv1  3 tiles x N = 64 / 32;  conv2  2 tiles x (18 / 6) x N = 96;  conv3  (54 / 18) x N = 32
// fc1 issues 1792 x 256 x 2 FLOP per board per product (3 / 1 products).  scripts/eval_kind_bench.py reads these four lines.
constexpr int TC_NUNIT_FLOP = 64 * 16 * 2;
constexpr int TC_CONV_NUNITS_NT2 = 3 * 64 + 2 * 18 * 96 + 54 * 32;   // 5376 -> 11.01 MFLOP per board
constexpr int TC_CONV_NUNITS_NT1 = 3 * 32 + 2 * 6 * 96 + 18 * 32;    // 1824 -> 3.74 MFLOP per board
constexpr int TC_FC_FLOP_PER_PRODUCT = 1792 * 256 * 2;                // x3 -> 2.75 MFLOP, x1 -> 0.92 MFLOP per board

struct TcWeights {
    const uint8_t *wc1;         // TCC_W1BYTES
    const uint8_t *wc2, *wc3;   // TCC_WBYTES each, already in the shared-memory layout
    const uint8_t *wfc;         // [split 2][k16 block 112][chunk 2][n 256][16 B]
};

// act3 in HBM, FC-tile layout: [split][tile of 128 rows][k chunk 224][row 128][8 fp16], k' = (y*4 + x)*32 + c
__device__ __forceinline__ size_t act3_off(int split, int n_tiles, int ridx, int kchunk) {
    return ((((size_t)split * n_tiles + (ridx >> 7)) * ACT3_KCHUNKS + kchunk) * 128 + (ridx & 127)) * 16;
}

// conv2 on one 64-row tile = 18 wgmma of N = 96: for each (dy, channel half): a1*W1, a1*W2, a2*W1 into the same 96 columns
// (NT = 1: a1*W1 only, 6 wgmma).
template <int NT>
__device__ __forceinline__ void issue_conv2(float (&d)[48], uint32_t a_addr, uint32_t w_addr) {
    const uint64_t a0 = gmma_desc(a_addr, TCC_R * 16, 128), b0 = gmma_desc(w_addr, 96 * 16, 128);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t a_hi = 2 * h * TCC_R + dy * 8, a_lo = a_hi + 4 * TCC_R;          // 16-byte units
            const uint32_t b_hi = (dy * 2 + h) * (TCC_WBLOCK / 16), b_lo = b_hi + 2 * 96;
            wgmma_n96(d, a0 + a_hi, b0 + b_hi, (dy | h) ? 1u : 0u);
            if (NT == 2) {
                wgmma_n96(d, a0 + a_hi, b0 + b_lo, 1u);
                wgmma_n96(d, a0 + a_lo, b0 + b_hi, 1u);
            }
        }
    }
}

// conv3 on its one 64-row tile = 3 accumulators x 18 wgmma of N = 32: for each (dy, channel half) and each dx, a1*W1, a1*W2, a2*W1
// (NT = 1: a1*W1 only, 3 x 6 wgmma).  The A operand of tap (dy, dx) starts 16 dx + dy rows (16-byte units) into act2.
template <int NT>
__device__ __forceinline__ void issue_conv3(float (&d)[3][16], uint32_t a_addr, uint32_t w_addr) {
    const uint64_t a0 = gmma_desc(a_addr, TCC_R2 * 16, 128), b0 = gmma_desc(w_addr, 32 * 16, 128);
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const uint32_t a_hi = 2 * h * TCC_R2 + 16 * dx + dy, a_lo = a_hi + TCC_A2SPLIT / 16;    // 16-byte units
                const uint32_t b_hi = ((dx * 3 + dy) * 2 + h) * 2 * (TCC_W3BLOCK / 16), b_lo = b_hi + TCC_W3BLOCK / 16;
                wgmma_n32(d[dx], a0 + a_hi, b0 + b_hi, (dy | h) ? 1u : 0u);
                if (NT == 2) {
                    wgmma_n32(d[dx], a0 + a_hi, b0 + b_lo, 1u);
                    wgmma_n32(d[dx], a0 + a_lo, b0 + b_hi, 1u);
                }
            }
        }
    }
}

// the conv1 operand of one board: row p = y*8 + x of the 18x8 output grid, k = tap = dy*3 + dx (fp16, exact {-1,0,1});
// taps 0..7 as ONE 16-byte store, tap 8 in the second k chunk
__device__ __forceinline__ void build_im2col3(uint8_t *im, const uint32_t *tab, int wt) {
    for (int p = wt; p < TCC_R; p += 128) {
        const int y = p >> 3, x = p & 7;
        uint32_t hv[9];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const uint32_t rw = tab[y + dy] >> x;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx)       // 1 settled, -1 falling piece, 0 empty (model_vv.py:212)
                hv[dy * 3 + dx] = ((rw >> dx) & 1u) * 0x3C00u | ((rw >> (16 + dx)) & 1u) * 0xBC00u;
        }
        *reinterpret_cast<uint4 *>(im + p * 16) =
            make_uint4(hv[0] | (hv[1] << 16), hv[2] | (hv[3] << 16), hv[4] | (hv[5] << 16), hv[6] | (hv[7] << 16));   // taps 0..7
        *reinterpret_cast<uint32_t *>(im + TCC_IMROWS * 16 + p * 16) = hv[8];                                        // tap 8
    }
}

// Test export of the activations that never leave shared memory: with DBG, each board's act1 and act2 slots are copied verbatim to
// dbg + ridx * TCC_DBG_BYTES once their epilogue has finished (b200_debug_tc_acts decodes them).  Only k_tc_conv_dbg instantiates it.
constexpr int TCC_DBG_BYTES = TCC_ASLOT + TCC_A2SLOT;
__device__ __forceinline__ void copy_slot(uint8_t *dst, const uint8_t *src, int bytes, int wt) {
    for (int i = wt; i < bytes / 16; i += 128) reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(src)[i];
}

template <int NT, bool DBG>
__device__ __forceinline__ void tc_conv_body(NetWeights W, TcWeights TW, const uint2 *req, const int32_t *n_req_ptr, const int32_t *first_ptr,
                                             const uint32_t *keys, int M, uint8_t *act3, int n_tiles, unsigned long long *prof, uint8_t *dbg) {
    extern __shared__ __align__(128) uint8_t smem[];
    float *sB = reinterpret_cast<float *>(smem + TCC_OFF_BIAS);
    const int t = threadIdx.x, wg = t >> 7, wt = t & 127, w = wt >> 5, lane = t & 31;
    // ---- one-time setup: weights into smem, zeroed operands (the im2col rows past 144 and act2 rows 96..97 stay zero)
    for (int i = t; i < TCC_WBYTES / 16; i += TCC_THREADS) {
        reinterpret_cast<uint4 *>(smem + TCC_OFF_W2)[i] = reinterpret_cast<const uint4 *>(TW.wc2)[i];
        reinterpret_cast<uint4 *>(smem + TCC_OFF_W3)[i] = reinterpret_cast<const uint4 *>(TW.wc3)[i];
    }
    for (int i = t; i < TCC_W1BYTES / 16; i += TCC_THREADS) reinterpret_cast<uint4 *>(smem + TCC_OFF_W1)[i] = reinterpret_cast<const uint4 *>(TW.wc1)[i];
    for (int i = t; i < (TCC_OFF_BIAS - TCC_OFF_A1) / 16; i += TCC_THREADS) reinterpret_cast<uint4 *>(smem + TCC_OFF_A1)[i] = make_uint4(0, 0, 0, 0);
    // relu(x * 2^-10 + b) * 16 == relu(fma(x, 2^-6, 16 b)) bit for bit (scaling by a power of two commutes with rounding): the biases
    // are kept pre-scaled and an epilogue value costs one fma + one max
    if (t < 32) { sB[t] = W.b1[t] * TC_SCALE_A; sB[32 + t] = W.b2[t] * TC_SCALE_A; sB[64 + t] = W.b3[t] * TC_SCALE_A; }
    fence_async_smem();
    __syncthreads();
    const int first = first_ptr ? *first_ptr : 0;      // this launch evaluates the requests [first, *n_req_ptr) (the deep lane's: see k_merge_requests)
    const int n_req = *n_req_ptr - first;
    // boards are handed out in runs of TCC_RUN consecutive requests (neighbouring act3 rows get written close in time)
    const int n_workers = (int)gridDim.x * TCC_WGS, wid = (int)blockIdx.x * TCC_WGS + wg;
    const int n_runs = (n_req + TCC_RUN - 1) / TCC_RUN;
    int n_local = 0;
    for (int run = wid; run < n_runs; run += n_workers) n_local += min(TCC_RUN, n_req - run * TCC_RUN);
    auto board_of = [&](int i) -> int { return first + ((i / TCC_RUN) * n_workers + wid) * TCC_RUN + (i % TCC_RUN); };
    uint8_t *act = smem + TCC_OFF_A1 + wg * TCC_ASLOT, *act2 = smem + TCC_OFF_A2 + wg * TCC_A2SLOT, *im = smem + TCC_OFF_IM + wg * TCC_IMSLOT;
    uint32_t *sKey = reinterpret_cast<uint32_t *>(smem + TCC_OFF_KEY) + wg * 32;
    const uint32_t s_act = smem_u32(act), s_act2 = smem_u32(act2), s_im = smem_u32(im);
    const uint32_t s_w1 = smem_u32(smem + TCC_OFF_W1), s_w2 = smem_u32(smem + TCC_OFF_W2), s_w3 = smem_u32(smem + TCC_OFF_W3);
    const int qd = lane & 3, rl = lane >> 2;             // accumulator rows 16w + rl (+8), columns 8j + 2qd (+1)
    constexpr float K23 = TC_UNSCALE * TC_SCALE_A, K1 = TC_SCALE_A / TC_SCALE_W;
    constexpr int SPLIT = 4 * TCC_R * 16;                // act1: second fp16 term
    const bool do_prof = prof && blockIdx.x == 0 && t == 0;
    long long pacc[4] = {0, 0, 0, 0}, ptick = clock64();
    auto prof_t = [&](int k) { if (do_prof) { const long long n = clock64(); pacc[k] += n - ptick; ptick = n; } };
    // A key is a random 48-byte read from an arena of tens of GB: lanes 0..11 of warp 0 fetch the NEXT board's key while this one is evaluated
    auto fetch = [&](int i) -> uint32_t {
        if (i >= n_local || lane >= 12) return 0u;
        const uint2 rq = req[board_of(i)];
        return keys[((size_t)rq.x * M + (rq.y & 0x0fffffffu)) * KEY_WORDS + lane];
    };
    uint32_t kw = w == 0 ? fetch(0) : 0u;
    for (int i = 0; i < n_local; ++i) {
        const int ridx = board_of(i);
        if (w == 0) {
            // row table: lane r < 20 holds board row r: settled cells in bits 0..9, the falling piece's cells in bits 16..25
            const uint32_t rowpair = __shfl_sync(0xffffffffu, kw, (lane >> 1) & 15), pcs = __shfl_sync(0xffffffffu, kw, 10);
            uint32_t tab = (rowpair >> ((lane & 1) * 16)) & 0x3ffu;
#pragma unroll
            for (int k = 0; k < 4; ++k) {                        // the falling piece's cells (sorted bytes of key word 10)
                const uint32_t cell = (pcs >> (8 * k)) & 0xffu, pr = (cell * 205u) >> 11, pcol = cell - pr * 10u;
                tab |= (pr == (uint32_t)lane ? 1u : 0u) << (16 + pcol);
            }
            kw = fetch(i + 1);
            if (lane < 20) sKey[lane] = tab;
        }
        wg_sync(wg);                                             // also: every warp has waited for the previous board's last MMAs
        build_im2col3(im, sKey, wt);
        fence_async_smem();
        wg_sync(wg);
        prof_t(0);
        // ---- conv1 (model_vv.py:32): im2col [192 x 16] x W1 [16 x 64] in three 64-row tiles; epilogue: bias + ReLU + split -> act1
        // (NT = 1: x W1 [16 x 32], the first weight term only; epilogue rounds to one fp16)
#pragma unroll 1
        for (int mt = 0; mt < 3; ++mt) {
            float d[16 * NT];
#pragma unroll
            for (int k = 0; k < 16 * NT; ++k) d[k] = 0.f;
            wgmma_fence();
            const uint64_t ad = gmma_desc(s_im + mt * 1024, TCC_IMROWS * 16, 128), bd = gmma_desc(s_w1, 64 * 16, 128);
            if constexpr (NT == 2) wgmma_n64(d, ad, bd, 0u);
            else wgmma_n32(d, ad, bd, 0u);                       // cout 0..31 of each k chunk: the first weight term
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(d);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = mt * 64 + 16 * w + 8 * h + rl;
                if (r < TCC_R) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {                // cout 8j + 2qd + e: weight split 1 sits 32 columns (4 blocks) further
                        const int c = 8 * j + 2 * qd;
                        uint8_t *dst = act + (j * TCC_R + r) * 16 + qd * 4;
                        if constexpr (NT == 2) {
                            const float o0 = fmaxf(fmaf(d[4 * (j + 4) + 2 * h] + d[4 * j + 2 * h], K1, sB[c]), 0.f);
                            const float o1 = fmaxf(fmaf(d[4 * (j + 4) + 2 * h + 1] + d[4 * j + 2 * h + 1], K1, sB[c + 1]), 0.f);
                            uint32_t hi, lo;
                            split2(o0, o1, hi, lo);
                            *reinterpret_cast<uint32_t *>(dst) = hi;
                            *reinterpret_cast<uint32_t *>(dst + SPLIT) = lo;
                        } else {
                            const float o0 = fmaxf(fmaf(d[4 * j + 2 * h], K1, sB[c]), 0.f);
                            const float o1 = fmaxf(fmaf(d[4 * j + 2 * h + 1], K1, sB[c + 1]), 0.f);
                            *reinterpret_cast<uint32_t *>(dst) = round1(o0, o1);
                        }
                    }
                }
            }
        }
        fence_async_smem();
        wg_sync(wg);
        prof_t(1);
        if constexpr (DBG) copy_slot(dbg + (size_t)ridx * TCC_DBG_BYTES, act, TCC_ASLOT, wt);
        // ---- conv2 (model_vv.py:34) on act1 (18x8 grid) -> act2 (column-major, its own buffer: tile 0's outputs reach row 87 of act2
        // while tile 1 still reads act1 rows 64..143)
#pragma unroll 1
        for (int mt = 0; mt < 2; ++mt) {
            float d[48];
#pragma unroll
            for (int k = 0; k < 48; ++k) d[k] = 0.f;
            wgmma_fence();
            issue_conv2<NT>(d, s_act + mt * 1024, s_w2);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(d);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int y = mt * 8 + 2 * w + h, x = rl;
                constexpr int NW = 4 * NT;                       // words per pixel and lane
                uint32_t v[NW];                                  // v[j + 4s]: channels 8j + 2qd (+1), fp16 term s
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {                // out[p] = D'[p][dx=0] + D'[p+1][dx=1] + D'[p+2][dx=2]
                        const int k = 4 * j + 2 * h + e;
                        const float s1 = __shfl_down_sync(0xffffffffu, d[16 + k], 4), s2 = __shfl_down_sync(0xffffffffu, d[32 + k], 8);
                        o[e] = fmaxf(fmaf((s2 + s1) + d[k], K23, sB[32 + 8 * j + 2 * qd + e]), 0.f);
                    }
                    if constexpr (NT == 2) split2(o[0], o[1], v[j], v[4 + j]);
                    else v[j] = round1(o[0], o[1]);
                }
                // Store k of lane (x, qd) writes word i = (k + x) & 7 at split i/4, chunk i%4, row x*16 + y: in 4-byte banks that is
                // (8 (i%4) + 4 (i/4) + 4y + qd) mod 32 (row x*16 is 256 B, a multiple of the 128-B bank line), so the six pixels x < 6
                // hit six disjoint 4-bank groups: one wavefront per store instead of a 6-way conflict.  The words are rotated into place
                // by x with selects (a dynamically indexed array would live in local memory).  NT = 1 rotates its four words by x & 3:
                // pixels x and x + 4 share a bank group, two wavefronts for each of four stores.
#pragma unroll
                for (int b = 1; b < NW; b <<= 1) {
                    uint32_t r[NW];
#pragma unroll
                    for (int k = 0; k < NW; ++k) r[k] = (x & b) ? v[(k + b) & (NW - 1)] : v[k];
#pragma unroll
                    for (int k = 0; k < NW; ++k) v[k] = r[k];
                }
                if (x < 6) {                                     // act2: 16x6 valid pixels
#pragma unroll
                    for (int k = 0; k < NW; ++k) {
                        const int i = (k + x) & (NW - 1);
                        *reinterpret_cast<uint32_t *>(act2 + (i >> 2) * TCC_A2SPLIT + ((i & 3) * TCC_R2 + x * 16 + y) * 16 + qd * 4) = v[k];
                    }
                }
            }
        }
        fence_async_smem();
        wg_sync(wg);
        prof_t(2);
        if constexpr (DBG) copy_slot(dbg + (size_t)ridx * TCC_DBG_BYTES + TCC_ASLOT, act2, TCC_A2SLOT, wt);
        // ---- conv3 (:36) on act2: one tile, warp w holds column x = w, lane rows y = 8h + rl; act3 -> HBM
        {
            float d[3][16];
#pragma unroll
            for (int k = 0; k < 16; ++k) d[0][k] = d[1][k] = d[2][k] = 0.f;
            wgmma_fence();
            issue_conv3<NT>(d, s_act2, s_w3);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(d[0]); fence_regs(d[1]); fence_regs(d[2]);
            const int x = w;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int y = 8 * h + rl;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int k = 4 * j + 2 * h + e;
                        o[e] = fmaxf(fmaf((d[2][k] + d[1][k]) + d[0][k], K23, sB[64 + 8 * j + 2 * qd + e]), 0.f);
                    }
                    if constexpr (NT == 2) {
                        uint32_t hi, lo;
                        split2(o[0], o[1], hi, lo);
                        if (y < 14) {
                            const int kc = (y * 4 + x) * 4 + j;
                            *reinterpret_cast<uint32_t *>(act3 + act3_off(0, n_tiles, ridx, kc) + qd * 4) = hi;
                            *reinterpret_cast<uint32_t *>(act3 + act3_off(1, n_tiles, ridx, kc) + qd * 4) = lo;
                        }
                    } else {
                        const uint32_t hi = round1(o[0], o[1]);
                        if (y < 14) *reinterpret_cast<uint32_t *>(act3 + act3_off(0, n_tiles, ridx, (y * 4 + x) * 4 + j) + qd * 4) = hi;
                    }
                }
            }
        }
        wg_sync(wg);
        prof_t(3);
    }
    if (do_prof) for (int k = 0; k < 4; ++k) atomicAdd(&prof[k], (unsigned long long)pacc[k]);
}

template <int NT>
__global__ void __launch_bounds__(TCC_THREADS, 1)
k_tc_conv(NetWeights W, TcWeights TW, const uint2 *req, const int32_t *n_req_ptr, const int32_t *first_ptr, const uint32_t *keys, int M, uint8_t *act3,
          int n_tiles, unsigned long long *prof) {
    tc_conv_body<NT, false>(W, TW, req, n_req_ptr, first_ptr, keys, M, act3, n_tiles, prof, nullptr);
}
template <int NT>
__global__ void __launch_bounds__(TCC_THREADS, 1)
k_tc_conv_dbg(NetWeights W, TcWeights TW, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, uint8_t *act3, int n_tiles, uint8_t *dbg) {
    tc_conv_body<NT, true>(W, TW, req, n_req_ptr, nullptr, keys, 0, act3, n_tiles, nullptr, dbg);
}

// ---------------------------------------------------------------------------------------------------- fc kernel
constexpr int TCF_CONSUMERS = 2;            // warpgroups 0-1: MMA + epilogue, 64 rows of the 128-row tile each
constexpr int TCF_PRODUCER = TCF_CONSUMERS * 4;   // warp 8: bulk copies
constexpr int TCF_THREADS = TCF_CONSUMERS * 128 + 32;
constexpr int TCF_STAGES = 8;
constexpr int TCF_A_BYTES = 2 * 128 * 16;   // one split of one k16 block of the A tile
constexpr int TCF_B_BYTES = 2 * 256 * 16;
constexpr int TCF_STAGE = 2 * TCF_A_BYTES + 2 * TCF_B_BYTES;   // 24576
constexpr int TCF_KBLOCKS = 112;            // 1792 / 16
constexpr int TCF_OFF_BAR = TCF_STAGES * TCF_STAGE;
constexpr int TCF_OFF_EPI = TCF_OFF_BAR + 256;                 // bias[256] | wout[2][256] | bout/ub/lb
static_assert(2 * TCF_STAGES * 8 <= 256, "barrier block overflows into the epilogue constants");
constexpr int TCF_SMEM = TCF_OFF_EPI + (256 * 3 + 8) * 4;
static_assert(TCF_SMEM <= 227 * 1024, "k_tc_fc shared memory");

// With DBG, each board's raw fp32 fc1 accumulator (before the 2^-10, the bias and the ReLU) is also written to dbg + ridx * 256, in torch
// column order (b200_debug_tc_acts returns it).  Only k_tc_fc_dbg instantiates it.
template <int NT, bool DBG>
__device__ __forceinline__ void tc_fc_body(NetWeights W, TcWeights TW, const uint8_t *act3, int n_tiles_alloc, const uint2 *req, const int32_t *n_req_ptr,
                                           float2 *eval_out, float *dbg) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + TCF_OFF_BAR);     // [stage] operands landed
    uint64_t *empty = full + TCF_STAGES;                                    // [stage] operands consumed (one arrival per consumer warpgroup)
    float *sBias = reinterpret_cast<float *>(smem + TCF_OFF_EPI), *sWo = sBias + 256, *sTail = sWo + 512;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    for (int i = t; i < 256; i += TCF_THREADS) { sBias[i] = W.bfc1[i]; sWo[i] = W.wout[i]; sWo[256 + i] = W.wout[256 + i]; }
    if (t < 2) { sTail[t] = W.bout[t]; sTail[2 + t] = W.ub[t]; sTail[4 + t] = W.lb[t]; }
    if (t == 0) {
        for (int i = 0; i < TCF_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TCF_CONSUMERS); }
        fence_barrier_init();
    }
    __syncthreads();
    const int n_req = *n_req_ptr;
    const int n_tiles = (n_req + 127) >> 7;
    if (warp == TCF_PRODUCER) {
        if (lane == 0) {   // ===== producer: bulk copies of the pre-laid-out operand blocks
            int stage = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                for (int j = 0; j < TCF_KBLOCKS; ++j) {
                    mbar_wait(&empty[stage], ph ^ 1);
                    mbar_expect_tx(&full[stage], NT * (TCF_A_BYTES + TCF_B_BYTES));
                    uint8_t *dst = smem + stage * TCF_STAGE;
#pragma unroll
                    for (int s = 0; s < NT; ++s) {               // NT = 1: the first term of each operand; its second-term slots stay unused
                        bulk_g2s(dst + s * TCF_A_BYTES, act3 + (((size_t)s * n_tiles_alloc + tile) * ACT3_KCHUNKS + 2 * j) * 2048, TCF_A_BYTES, &full[stage]);
                        bulk_g2s(dst + 2 * TCF_A_BYTES + s * TCF_B_BYTES, TW.wfc + ((size_t)s * TCF_KBLOCKS + j) * TCF_B_BYTES, TCF_B_BYTES, &full[stage]);
                    }
                    if (++stage == TCF_STAGES) { stage = 0; ph ^= 1; }
                }
            }
        }
    } else {   // ===== consumers: D[64 x 256] += A[64 x 16] * B[256 x 16]^T per warpgroup, three split terms per k block (NT = 1: one)
        const int wg = t >> 7, w = warp & 3, qd = lane & 3, rl = lane >> 2;
        constexpr int T0 = NT == 2 ? 0 : 2;              // first of the three products issued
        int stage = 0; uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            float d[128];
#pragma unroll
            for (int k = 0; k < 128; ++k) d[k] = 0.f;
            int prev = -1;
            for (int j = 0; j < TCF_KBLOCKS; ++j) {
                mbar_wait(&full[stage], ph);
                const uint32_t sbase = smem_u32(smem + stage * TCF_STAGE);
                wgmma_fence();
#pragma unroll
                for (int term = T0; term < 3; ++term) {  // a1*b2, a2*b1, a1*b1 (small terms first); NT = 1: a1*b1
                    const int sa = term == 1 ? 1 : 0, sb = term == 0 ? 1 : 0;
                    const uint64_t ad = gmma_desc(sbase + sa * TCF_A_BYTES + wg * 1024, 128 * 16, 128);
                    const uint64_t bd = gmma_desc(sbase + 2 * TCF_A_BYTES + sb * TCF_B_BYTES, 256 * 16, 128);
                    wgmma_n256(d, ad, bd, (j > 0 || term > T0) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();                         // the previous k block's MMAs are done with their stage
                if (prev >= 0 && (t & 127) == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == TCF_STAGES) { stage = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(d);
            if constexpr (DBG) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ridx = tile * 128 + wg * 64 + 16 * w + 8 * h + rl;
                    if (ridx < n_req)
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            dbg[(size_t)ridx * 256 + 8 * j + 2 * qd] = d[4 * j + 2 * h];
                            dbg[(size_t)ridx * 256 + 8 * j + 2 * qd + 1] = d[4 * j + 2 * h + 1];
                        }
                }
            }
            if ((t & 127) == 0) mbar_arrive(&empty[prev]);
            float p0[2] = {0.f, 0.f}, p1[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < 32; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * j + 2 * qd + e;
                        const float hv = fmaxf(d[4 * j + 2 * h + e] * TC_UNSCALE + sBias[c], 0.f);   // model_vv.py:39-40
                        p0[h] = fmaf(hv, sWo[c], p0[h]); p1[h] = fmaf(hv, sWo[256 + c], p1[h]);      // :41
                    }
#pragma unroll
            for (int h = 0; h < 2; ++h) {                // the four lanes of a row hold interleaved column quarters
                p0[h] += __shfl_xor_sync(0xffffffffu, p0[h], 1); p1[h] += __shfl_xor_sync(0xffffffffu, p1[h], 1);
                p0[h] += __shfl_xor_sync(0xffffffffu, p0[h], 2); p1[h] += __shfl_xor_sync(0xffffffffu, p1[h], 2);
                const int ridx = tile * 128 + wg * 64 + 16 * w + 8 * h + rl;
                if (qd == 0 && ridx < n_req) {
                    const float x0 = p0[h] + sTail[0], x1 = p1[h] + sTail[1];
                    const float s0 = 1.f / (1.f + expf(-x0)), s1 = 1.f / (1.f + expf(-x1));      // :42
                    const uint2 rq = req[ridx];
                    eval_out[(size_t)rq.x * 8 + (rq.y >> 28)] =
                        make_float2(__fadd_rn(__fmul_rn(s0, sTail[2]), sTail[4]), __fadd_rn(__fmul_rn(s1, sTail[3]), sTail[5]));   // :51
                }
            }
        }
    }
}

template <int NT>
__global__ void __launch_bounds__(TCF_THREADS, 1)
k_tc_fc(NetWeights W, TcWeights TW, const uint8_t *act3, int n_tiles_alloc, const uint2 *req, const int32_t *n_req_ptr, float2 *eval_out) {
    tc_fc_body<NT, false>(W, TW, act3, n_tiles_alloc, req, n_req_ptr, eval_out, nullptr);
}
template <int NT>
__global__ void __launch_bounds__(TCF_THREADS, 1)
k_tc_fc_dbg(NetWeights W, TcWeights TW, const uint8_t *act3, int n_tiles_alloc, const uint2 *req, const int32_t *n_req_ptr, float2 *eval_out,
            float *dbg) {
    tc_fc_body<NT, true>(W, TW, act3, n_tiles_alloc, req, n_req_ptr, eval_out, dbg);
}

// ---------------------------------------------------------------------------------------------------- host side
struct TcState {
    uint8_t *d_w = nullptr;      // wc1 | wc2 | wc3 | wfc
    TcWeights TW{};
    uint8_t *d_act3 = nullptr; size_t tiles = 0;
};

static inline void host_split2(float x, uint16_t *o) {   // x*scale = h1 + h2 in fp16
    __half h1 = __float2half_rn(x);
    __half h2 = __float2half_rn(x - __half2float(h1));
    memcpy(&o[0], &h1, 2); memcpy(&o[1], &h2, 2);
}
static inline float host_half_f(uint16_t h) { __half x; memcpy(&x, &h, 2); return __half2float(x); }

// The split scales a weight by TC_SCALE_W before rounding it to fp16: |w| * 64 above fp16's largest finite value (65504, |w| >= ~1023.5)
// would become an infinity and poison every output.  True when every weight the split carries (conv1-3, fc1) is in range (NaN is not).
static inline bool tc_split_fits(const float *x, size_t n) {
    for (size_t i = 0; i < n; ++i)
        if (!(fabsf(x[i]) * TC_SCALE_W <= 65504.f)) return false;
    return true;
}
static bool tc_weights_fit(const float *w) {
    const float *c1w = w, *c2w = w + 288 + 32, *c3w = c2w + 9216 + 32, *f1w = c3w + 9216 + 32;
    return tc_split_fits(c1w, 288) && tc_split_fits(c2w, 9216) && tc_split_fits(c3w, 9216) && tc_split_fits(f1w, (size_t)256 * 1792);
}

// w = the state_dict-order weight vector of include/b200_tetris_mcts.h.  Pure re-layout + fp16 splitting.
static int tc_prepare(void **state, const float *w, cudaStream_t stream) {
    TcState *st = (TcState *)*state;
    if (!st) { st = new TcState(); *state = st; }
    const float *c1w = w, *c2w = w + 288 + 32, *c3w = c2w + 9216 + 32, *f1w = c3w + 9216 + 32;
    const size_t fc_bytes = (size_t)2 * TCF_KBLOCKS * TCF_B_BYTES;
    std::vector<uint8_t> h(TCC_W1BYTES + 2 * (size_t)TCC_WBYTES + fc_bytes);
    uint16_t *p1 = reinterpret_cast<uint16_t *>(h.data());
    uint16_t *p2 = reinterpret_cast<uint16_t *>(h.data() + TCC_W1BYTES), *p3 = reinterpret_cast<uint16_t *>(h.data() + TCC_W1BYTES + TCC_WBYTES);
    uint16_t *pf = reinterpret_cast<uint16_t *>(h.data() + TCC_W1BYTES + 2 * (size_t)TCC_WBYTES);
    for (int c2 = 0; c2 < 2; ++c2)                               // conv1: [chunk][n = split*32 + cout][8], k = tap
        for (int n = 0; n < 32; ++n)
            for (int e = 0; e < 8; ++e) {
                const int tap = 8 * c2 + e;
                uint16_t s2[2] = {0, 0};
                if (tap < 9) host_split2(c1w[n * 9 + tap] * TC_SCALE_W, s2);
                for (int s = 0; s < 2; ++s) p1[((size_t)c2 * 64 + s * 32 + n) * 8 + e] = s2[s];
            }
    for (int dy = 0; dy < 3; ++dy)
        for (int hh = 0; hh < 2; ++hh)
            for (int c2 = 0; c2 < 2; ++c2)
                for (int dx = 0; dx < 3; ++dx)
                    for (int n = 0; n < 32; ++n)
                        for (int e = 0; e < 8; ++e) {
                            int ci = 16 * hh + 8 * c2 + e, tap = dy * 3 + dx;
                            uint16_t s2[2], s3[2];
                            host_split2(c2w[(n * 32 + ci) * 9 + tap] * TC_SCALE_W, s2);
                            host_split2(c3w[(n * 32 + ci) * 9 + tap] * TC_SCALE_W, s3);
                            for (int s = 0; s < 2; ++s) {
                                // conv2: [(dy, half)][split][chunk][n = dx*32 + cout][8] (dx stacked along N)
                                p2[(((((size_t)(dy * 2 + hh)) * 2 + s) * 2 + c2) * 96 + dx * 32 + n) * 8 + e] = s2[s];
                                // conv3: [(dx, dy, half)][split][chunk][cout][8] (one block per accumulator and A shift)
                                p3[((((((size_t)(dx * 3 + dy)) * 2 + hh) * 2 + s) * 2 + c2) * 32 + n) * 8 + e] = s3[s];
                            }
                        }
    for (int j = 0; j < TCF_KBLOCKS; ++j)
        for (int c2 = 0; c2 < 2; ++c2)
            for (int n = 0; n < 256; ++n)
                for (int e = 0; e < 8; ++e) {
                    int kp = j * 16 + c2 * 8 + e, p = kp >> 5, c = kp & 31;      // k' = pixel*32 + channel, pixel = y*4 + x
                    uint16_t s2[2];
                    host_split2(f1w[(size_t)n * 1792 + c * 56 + p] * TC_SCALE_W, s2);
                    for (int s = 0; s < 2; ++s) pf[((((size_t)s * TCF_KBLOCKS + j) * 2 + c2) * 256 + n) * 8 + e] = s2[s];
                }
    if (!st->d_w && cudaMalloc(&st->d_w, h.size()) != cudaSuccess) return 1;
    if (cudaMemcpyAsync(st->d_w, h.data(), h.size(), cudaMemcpyHostToDevice, stream) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return 1;
    st->TW.wc1 = st->d_w; st->TW.wc2 = st->d_w + TCC_W1BYTES; st->TW.wc3 = st->TW.wc2 + TCC_WBYTES; st->TW.wfc = st->TW.wc3 + TCC_WBYTES;
    if (cudaFuncSetAttribute(k_tc_conv<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCC_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_conv<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCC_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_conv_dbg<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCC_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_conv_dbg<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCC_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_fc<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCF_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_fc<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCF_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_fc_dbg<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCF_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tc_fc_dbg<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TCF_SMEM) != cudaSuccess) return 1;
    return 0;
}

static int tc_ensure_act3(TcState *st, size_t max_rows, cudaStream_t stream) {
    size_t tiles = (max_rows + 127) / 128;
    if (st->tiles >= tiles) return 0;
    if (st->d_act3) { cudaStreamSynchronize(stream); cudaFree(st->d_act3); st->d_act3 = nullptr; }
    size_t bytes = (size_t)2 * tiles * ACT3_KCHUNKS * 2048;
    if (cudaMalloc(&st->d_act3, bytes) != cudaSuccess) return 1;
    cudaMemsetAsync(st->d_act3, 0, bytes, stream);
    st->tiles = tiles;
    return 0;
}

static void tc_destroy(void *state) {
    TcState *st = (TcState *)state;
    if (!st) return;
    cudaFree(st->d_w); cudaFree(st->d_act3);
    delete st;
}

}  // namespace b200
