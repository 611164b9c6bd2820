// trainer.cu — the value-network training step of the reference on the GPU (SURVEY §8f.2), behind the C-ABI of include/b200_tetris_mcts.h.
//
// Reference (file:line in /root/reference):
//   Net.forward                    model/model_vv.py:13-52     conv3x3(1->32) ReLU conv3x3(32->32) ReLU conv3x3(32->32) ReLU flatten fc(1792->256) ReLU
//                                                              fc(256->2) sigmoid, * out_ubound + out_lbound
//   GaussianLL                     model/model_vv.py:94-101    logl = log(var_p) + ((mean - mean_p)^2 + var) / var_p - log(var) - 1
//   Model_VV._loss                 model/model_vv.py:136-153   variance.clamp_(min=1e-1); weighted: std_mean(weight * logl, unbiased=False)
//   Model.train                    model/model.py:95-119       zero_grad, loss.backward(), gradient norm, optional clip, optimizer.step()
//   Yogi.step                      model/yogi.py:39-90         (lr=1e-3, eps=1e-3, weight_decay=1e-3: model_vv.py:132)
//   Model_VV.train_data            model/model_vv.py:227-231   out_ubound <- [max(value), max(variance)] of the training data
//   Model.train_data               model/model.py:176-249      b200_trainer_train_rows_dev: a validation interval of steps on device rows, batches
//                                                              drawn on the device, one host synchronisation; _loss_rows_dev / b200_rows_stats_dev
//
// Arithmetic: fp32 storage as in the reference; every contraction (forward GEMMs, weight / bias / input gradients) accumulates in fp64 and
// rounds once to fp32, so the result does not depend on a blocking order and sits within the reference's own fp32 rounding noise
// (tests: rtol 1e-5 against goldens recorded from the reference's own Model_VV.train on torch CPU).  Convolutions are lowered to
// GEMMs through explicit im2col buffers in HBM (the PyTorch [co][ci][ky][kx] weight layout is used as it lies: k = ci*9 + ky*3 + kx).
// No atomics: every reduction has a fixed order, training is bit-reproducible run to run.
//
// Trainer kinds (b200_trainer_create_kind).  B200_TRAIN_FP64 runs every contraction through k_gemm (CUDA cores, fp64 accumulation, above).
// B200_TRAIN_TC runs the forward, input-gradient and conv / fc1 weight-gradient GEMMs through k_gemm_tc on Hopper tensor cores (wgmma
// m64nNk8 .f32.tf32.tf32); fc_out's 2 x 256 weight gradient, the bias sums and everything around the GEMMs are shared by both kinds.
// Precision of the tc kind (3xTF32):
//   - split: every fp32 operand x is stored as big = rna_tf32(x), small = rna_tf32(x - big) (x - big is exact in fp32).  tf32 keeps 10 + 1
//     mantissa bits and fp32's exponent range, so |x - big| <= 2^-11 |x|, |x - big - small| <= 2^-22 |x| down to fp32's subnormal floor:
//     nothing is pre-scaled and nothing underflows that fp32 itself would hold (gradients of 1e-30 keep 22 bits).  Below 2^-126 the terms
//     are subnormal and the split's error becomes absolute, <= 2^-137; above (2 - 2^-11) 2^127 (0.02 % below fp32's largest) big rounds
//     to infinity.
//   - products: a*b is accumulated as a_small*b_big + a_big*b_small + a_big*b_big (small products first, fp32 accumulators); the dropped
//     a_small*b_small and the two split residuals leave <= 3 * 2^-22 |a b| per product.
//   - reductions: the tensor core's fp32 accumulation does not round to nearest (measured on an H100: a 2048-k wgmma chain was biased by
//     ~1e-4 of the result on same-sign sums, consistent with truncating each addition), so a wgmma chain covers one 32-wide k tile only
//     (12 MMAs, scale-d = 0 at the tile's first): its sum goes into a separate fp32 register accumulator by an IEEE round-to-nearest FADD.
//     Truncation over 32 terms is <= 32 * 2^-23 = 4e-6 of the tile's |terms| worst case and ~2^-24 sqrt(32) typical; the FADD chain of
//     one chunk covers at most TG_KCHUNK = 2048 consecutive k (64 tiles): statistically ~sqrt(64) * 2^-24 = 5e-7 of the sum of |terms|
//     (worst case 64 * 2^-24 = 4e-6).  Longer reductions (the weight gradients reduce
//     over B * 56 .. B * 144 pixels, 590 k terms at B = 4096) are cut into chunks of <= 2048 k; each chunk writes its tile as an fp64
//     partial and k_finish adds the partials in ascending chunk order in fp64, so the error does not grow with the batch.  The chunk
//     length rests on the worst case: one FADD chain over all 590 k terms (18 k tile sums) is bounded only by 18k * 2^-24 = 1.1e-3 of
//     the |terms|, 2048 k by 4e-6, under the 1e-5 the trainer is held to (typical errors grow like sqrt(n) and stay below 1e-5 either
//     way on the tests' data, so no test separates the two).
//   - together: every GEMM output is within ~1e-6 of the sum of its |terms| (split, tile truncation and chunk sum; ~1e-5 worst case), the same class as the
//     inference split (valuenet_tc.cuh); tests hold loss, gradient norm and each gradient tensor to 1e-5 of float64 autograd.
//   - determinism: the chunking depends on the shapes alone and no reduction uses atomics: the tc kind is bit-reproducible run to run and
//     b200_trainer_train_rows_dev stays bit-identical to b200_trainer_step_rows_dev fed the same indices.
// B200_TRAIN_TF32 runs the same GEMMs through k_gemm_tf32 with one tf32 term per operand (one wgmma per k8, a third of the tc kind's):
//   - operands: x -> rna_tf32(x), |x - rna_tf32(x)| <= 2^-11 |x| (2^-137 absolute below fp32's normal range); the product of two
//     rounded operands (11 x 11 significant bits) is exact in the fp32 accumulator.
//   - reductions: the tc kind's structure unchanged (one wgmma chain per 32-wide k tile, round-to-nearest FADD into the chunk accumulator,
//     tc_k_per_split's k ranges, fp64 partials, k_finish), so per element a result is the exact sum of the rounded products within the
//     tc accumulation bound (32 instead of 96 truncating adds per tile), independent of the batch size.
//   - against float64: each GEMM output is within 2^-10 of its |term| sum from the two operand roundings, plus the accumulation; summed
//     to first order over the products on a result's path this holds the loss within 4 * 2^-10 and the gradient norm within 8 * 2^-10;
//     a gradient element is held to that error carried through the head (GaussianLL's mean - pred can cancel) and the backward pass in
//     absolute values (tests/test_gpu_trainer_tf32.py).  TF32 with one term is also what torch uses for the reference's conv layers on
//     Hopper by default (cudnn.allow_tf32).
//   - implicit im2col: the conv forward GEMMs gather A from the NHWC activations (k = ci*9 + ky*3 + kx), the conv weight gradients gather
//     col^T the same way, and the input gradients of conv3 / conv2 are one GEMM each writing da2 / da1 directly (k = (ky*3 + kx)*32 + co,
//     K = 288, taps outside dY are zero terms, ReLU mask in the epilogue): no col1-3 / dcol3 / dcol2 buffers and no k_col2im_relu.
//   - determinism: as the tc kind.
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200_tetris_mcts.h"
#include "gmma.cuh"

namespace {

thread_local std::string g_terr;
int tfail(int code, const std::string &msg) { g_terr = msg; return code; }
#define TCK(call)                                                                                         \
    do {                                                                                                  \
        cudaError_t _e = (call);                                                                          \
        if (_e != cudaSuccess) return tfail(B200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e)); \
    } while (0)

// state_dict order (include/b200_tetris_mcts.h B200_N_WEIGHTS)
constexpr int O_C1W = 0, O_C1B = 288, O_C2W = 320, O_C2B = 9536, O_C3W = 9568, O_C3B = 18784, O_F1W = 18816, O_F1B = 477568,
              O_FOW = 477824, O_FOB = 478336, O_UB = 478338, O_LB = 478340, N_TRAIN = 478338, N_ALL = 478342;
constexpr int N_TENSORS = 10;
const int T_OFF[N_TENSORS + 1] = {O_C1W, O_C1B, O_C2W, O_C2B, O_C3W, O_C3B, O_F1W, O_F1B, O_FOW, O_FOB, N_TRAIN};

// ------------------------------------------------------------------------------------------------ GEMM (fp32 in/out, fp64 accumulate)
// C[M,N] (+)= op(A)[M,K] * op(B)[K,N];  TA: A is stored [K][M] (transposed), else [M][K];  TB: B is stored [N][K], else [K][N].
// 64x64 tile, 16-wide k steps, 256 threads, 4x4 outputs per thread; k ascending inside a CTA.  split_k > 1: blockIdx.z takes k range z and
// writes its partial tile to C + z*M*N; k_reduce_splits adds the partials in ascending z (fixed order, fp64).
template <bool TA, bool TB>
__global__ void __launch_bounds__(256) k_gemm(const float *__restrict__ A, const float *__restrict__ B, double *__restrict__ Cpart,
                                              int M, int N, int K, int k_per_split, float *__restrict__ Cdirect, const float *__restrict__ bias, int relu) {
    __shared__ float sA[16][64 + 1], sB[16][64 + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    const int kb = blockIdx.z * k_per_split, ke = min(K, kb + k_per_split);
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    for (int k0 = kb; k0 < ke; k0 += 16) {
        for (int e = threadIdx.x; e < 16 * 64; e += 256) {
            int kk, mm;
            if (TA) { mm = e & 63; kk = e >> 6; } else { kk = e & 15; mm = e >> 4; }
            const int k = k0 + kk, m = m0 + mm;
            float v = 0.f;
            if (k < ke && m < M) v = TA ? A[(size_t)k * M + m] : A[(size_t)m * K + k];
            sA[kk][mm] = v;
        }
        for (int e = threadIdx.x; e < 16 * 64; e += 256) {
            int kk, nn;
            if (TB) { kk = e & 15; nn = e >> 4; } else { nn = e & 63; kk = e >> 6; }
            const int k = k0 + kk, n = n0 + nn;
            float v = 0.f;
            if (k < ke && n < N) v = TB ? B[(size_t)n * K + k] : B[(size_t)k * N + n];
            sB[kk][nn] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = (double)sA[kk][ty * 4 + i]; b[i] = (double)sB[kk][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    if (Cdirect) {          // one k range: round once to fp32, bias / ReLU here (no partial-sum buffer)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
                if (m < M && n < N) {
                    float v = (float)acc[i][j];
                    if (bias) v = v + bias[n];
                    if (relu) v = fmaxf(v, 0.f);
                    Cdirect[(size_t)m * N + n] = v;
                }
            }
        return;
    }
    double *C = Cpart + (size_t)blockIdx.z * M * N;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
            if (m < M && n < N) C[(size_t)m * N + n] = acc[i][j];
        }
}

// ------------------------------------------------------------------------------------------------ GEMM on tensor cores (3xTF32, the tc kind)
// C[M,N] (+)= op(A)[M,K] * op(B)[K,N] with k_gemm's TA / TB storage conventions; ct: C is stored transposed ([N][M]), which lets a
// 32-row weight gradient run as a 32-column product.  One warpgroup per CTA, a 64 x BN output tile, 32-wide k tiles.  The staging
// loads read the tile (transposed or not) into registers, split each value into two tf32 terms and store both K-major in shared
// memory in the no-swizzle core-matrix layout [k chunk of 4][row][16 B]: a k8 step is two chunks ROWS * 16 B apart (LBO), 8-row groups
// are 128 B apart (SBO).  The next tile's loads are in flight while the wgmmas of this one run.  blockIdx.z covers k range z; more than
// one range: each writes its fp32 tile as an fp64 partial to Cpart + z*M*N and k_finish sums them (see the file header).
constexpr int TG_BM = 64, TG_BK = 32, TG_KCHUNK = 2048;
static_assert(TG_KCHUNK % TG_BK == 0, "chunks are whole k tiles");

__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands from shared memory (K-major), fp32 accumulators in valuenet_tc.cuh's layout:
// thread t holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8j + 2*(t%4) (+1) in d[4j + {0,1}] (row) / d[4j + {2,3}] (row + 8).
// accumulate == 0 overwrites D.
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
        "}, %16, %17, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <bool TA, bool TB, int BN>
__global__ void __launch_bounds__(128) k_gemm_tc(const float *__restrict__ A, const float *__restrict__ B, double *__restrict__ Cpart,
                                                 int M, int N, int K, int k_per_split, float *__restrict__ Cdirect, const float *__restrict__ bias,
                                                 int relu, int ct) {
    static_assert(BN == 32 || BN == 64, "wgmma_tf32 covers N = 32 and 64");
    constexpr int NA = TG_BM * TG_BK / 128, NB = BN * TG_BK / 128, KC = TG_BK / 4;
    __shared__ __align__(128) float sA[2][KC][TG_BM][4];     // [big / small][k chunk][row][4 k]
    __shared__ __align__(128) float sB[2][KC][BN][4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * TG_BM, n0 = blockIdx.x * BN;
    const int kb = blockIdx.z * k_per_split, ke = min(K, kb + k_per_split);
    // element i of a thread's share of the A / B tile: (row, k) chosen so that a warp reads along the stored fast index
    auto a_at = [&](int i, int &mm, int &kk) { const int e = i * 128 + tid; if (TA) { mm = e & 63; kk = e >> 6; } else { kk = e & 31; mm = e >> 5; } };
    auto b_at = [&](int i, int &nn, int &kk) { const int e = i * 128 + tid; if (TB) { kk = e & 31; nn = e >> 5; } else { nn = e % BN; kk = e / BN; } };
    float ra[NA], rb[NB];
    auto load = [&](int k0) {
#pragma unroll
        for (int i = 0; i < NA; ++i) {
            int mm, kk; a_at(i, mm, kk);
            const int k = k0 + kk, m = m0 + mm;
            ra[i] = (k < ke && m < M) ? (TA ? A[(size_t)k * M + m] : A[(size_t)m * K + k]) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            int nn, kk; b_at(i, nn, kk);
            const int k = k0 + kk, n = n0 + nn;
            rb[i] = (k < ke && n < N) ? (TB ? B[(size_t)n * K + k] : B[(size_t)k * N + n]) : 0.f;
        }
    };
    float d[BN / 2], acc[BN / 2];                          // d: this k tile's sum (tensor core), acc: the chunk's sum (FADD, round to nearest)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { d[i] = 0.f; acc[i] = 0.f; }
    const uint32_t sa = b200::smem_u32(&sA[0][0][0][0]), sb = b200::smem_u32(&sB[0][0][0][0]);
    constexpr uint32_t A_TERM = KC * TG_BM * 16, B_TERM = KC * BN * 16;     // bytes of one split term
    load(kb);
    for (int k0 = kb; k0 < ke; k0 += TG_BK) {
        __syncthreads();                                   // the previous tile's wgmmas are complete (every thread waited on them)
#pragma unroll
        for (int i = 0; i < NA; ++i) {
            int mm, kk; a_at(i, mm, kk);
            const float big = tf32_rna(ra[i]);
            sA[0][kk >> 2][mm][kk & 3] = big;
            sA[1][kk >> 2][mm][kk & 3] = tf32_rna(ra[i] - big);
        }
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            int nn, kk; b_at(i, nn, kk);
            const float big = tf32_rna(rb[i]);
            sB[0][kk >> 2][nn][kk & 3] = big;
            sB[1][kk >> 2][nn][kk & 3] = tf32_rna(rb[i] - big);
        }
        b200::fence_async_smem();
        __syncthreads();
        b200::wgmma_fence();
#pragma unroll
        for (int s = 0; s < TG_BK / 8; ++s) {              // a_small*b_big, a_big*b_small, a_big*b_big (small products first)
            const uint32_t ao = s * 2 * TG_BM * 16, bo = s * 2 * BN * 16;
            wgmma_tf32(d, b200::gmma_desc(sa + A_TERM + ao, TG_BM * 16, 128), b200::gmma_desc(sb + bo, BN * 16, 128), s ? 1u : 0u);
            wgmma_tf32(d, b200::gmma_desc(sa + ao, TG_BM * 16, 128), b200::gmma_desc(sb + B_TERM + bo, BN * 16, 128), 1u);
            wgmma_tf32(d, b200::gmma_desc(sa + ao, TG_BM * 16, 128), b200::gmma_desc(sb + bo, BN * 16, 128), 1u);
        }
        b200::wgmma_commit();
        if (k0 + TG_BK < ke) load(k0 + TG_BK);            // next tile's global loads overlap this tile's MMAs
        b200::wgmma_wait<0>();
        b200::fence_regs(d);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += d[i];
    }
    const int w = tid >> 5, lane = tid & 31, qd = lane & 3, rl = lane >> 2;
    double *Cp = Cdirect ? nullptr : Cpart + (size_t)blockIdx.z * M * N;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = m0 + 16 * w + 8 * h + rl, n = n0 + 8 * j + 2 * qd + e;
                if (m >= M || n >= N) continue;
                const size_t o = ct ? (size_t)n * M + m : (size_t)m * N + n;
                const float a = acc[4 * j + 2 * h + e];
                if (Cdirect) {                             // one k range: bias / ReLU here (no partial-sum buffer)
                    float v = a;
                    if (bias) v = v + bias[n];
                    if (relu) v = fmaxf(v, 0.f);
                    Cdirect[o] = v;
                } else {
                    Cp[o] = (double)a;
                }
            }
}

// ------------------------------------------------------------------------------------------------ GEMM on tensor cores (one tf32 term, the tf32 kind)
// k_gemm_tc with one term per operand: each fp32 operand is stored as rna_tf32(x) and each k8 step is one wgmma; the k tiles, the FADD
// chunk accumulator, the k ranges (tc_k_per_split), the fp64 partials and the epilogue are k_gemm_tc's.  The operands are read through
// the accessor AOP / BOP names, so a convolution needs no im2col or col2im buffer:
//   OP_N, OP_T   A stored [M][K] / [K][M], B stored [K][N] / [N][K] (k_gemm's TA / TB)
//   OP_CONV      A[m][k] = im2col(act)[m][k]: m = (b, y, x) an output pixel of the valid 3x3 conv of act [B][H][W][C] (NHWC),
//                k = ci*9 + ky*3 + kx (k_im2col's order)
//   OP_CONV_T    A[m][k] = im2col(act)[k][m] (a conv weight gradient's col^T)
//   OP_DGRAD     A[m][k] = dY[b][yy - ky][xx - kx][co] for the input pixel m = (b, yy, xx) of a conv whose output gradient dY is
//                [B][H-2][W-2][32]; k = (ky*3 + kx)*32 + co, so each 32-wide k tile is one tap; 0 where the tap falls outside dY
//   OP_DGRAD_W   B[k][n] = Wt[co][n][ky][kx] with OP_DGRAD's k (the layer's weight [32][C*9])
// H, W, C: the conv input's geometry, compile-time so that the index divisions are multiplications.  mask (one k range only): the output
// is mask[m][n] > 0 ? sum : 0 (the ReLU of the layer below, as k_col2im_relu).
enum { OP_N = 0, OP_T = 1, OP_CONV = 2, OP_CONV_T = 3, OP_DGRAD = 4, OP_DGRAD_W = 5 };

template <int H, int W, int C>
__device__ __forceinline__ float im2col_at(const float *__restrict__ act, int pix, int k) {
    constexpr int OH = H - 2, OW = W - 2;
    const int b = pix / (OH * OW), r = pix - b * (OH * OW), y = r / OW, x = r - y * OW;
    const int ci = k / 9, tap = k - ci * 9, ky = tap / 3, kx = tap - ky * 3;
    return act[(((size_t)b * H + y + ky) * W + x + kx) * C + ci];
}
template <int H, int W>
__device__ __forceinline__ float dgrad_at(const float *__restrict__ dy, int pix, int k) {
    constexpr int OH = H - 2, OW = W - 2;
    const int b = pix / (H * W), r = pix - b * (H * W), yy = r / W, xx = r - yy * W;
    const int tap = k >> 5, ky = tap / 3, y = yy - ky, x = xx - (tap - ky * 3);
    return (y >= 0 && y < OH && x >= 0 && x < OW) ? dy[(((size_t)b * OH + y) * OW + x) * 32 + (k & 31)] : 0.f;
}

template <int AOP, int BOP, int BN, int H, int W, int C>
__global__ void __launch_bounds__(128) k_gemm_tf32(const float *__restrict__ A, const float *__restrict__ B, double *__restrict__ Cpart,
                                                   int M, int N, int K, int k_per_split, float *__restrict__ Cdirect, const float *__restrict__ bias,
                                                   int relu, int ct, const float *__restrict__ mask) {
    static_assert(BN == 32 || BN == 64, "wgmma_tf32 covers N = 32 and 64");
    constexpr int NA = TG_BM * TG_BK / 128, NB = BN * TG_BK / 128, KC = TG_BK / 4;
    constexpr bool AM = AOP == OP_T || AOP == OP_CONV_T, BK = BOP == OP_T || BOP == OP_DGRAD_W;    // a warp's loads run along m / along k
    __shared__ __align__(128) float sA[KC][TG_BM][4];        // [k chunk][row][4 k]
    __shared__ __align__(128) float sB[KC][BN][4];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * TG_BM, n0 = blockIdx.x * BN;
    const int kb = blockIdx.z * k_per_split, ke = min(K, kb + k_per_split);
    auto a_at = [&](int i, int &mm, int &kk) { const int e = i * 128 + tid; if (AM) { mm = e & 63; kk = e >> 6; } else { kk = e & 31; mm = e >> 5; } };
    auto b_at = [&](int i, int &nn, int &kk) { const int e = i * 128 + tid; if (BK) { kk = e & 31; nn = e >> 5; } else { nn = e % BN; kk = e / BN; } };
    auto a_val = [&](int m, int k) -> float {
        if constexpr (AOP == OP_N) return A[(size_t)m * K + k];
        else if constexpr (AOP == OP_T) return A[(size_t)k * M + m];
        else if constexpr (AOP == OP_CONV) return im2col_at<H, W, C>(A, m, k);
        else if constexpr (AOP == OP_CONV_T) return im2col_at<H, W, C>(A, k, m);
        else return dgrad_at<H, W>(A, m, k);
    };
    auto b_val = [&](int k, int n) -> float {
        if constexpr (BOP == OP_N) return B[(size_t)k * N + n];
        else if constexpr (BOP == OP_T) return B[(size_t)n * K + k];
        else return B[(size_t)(k & 31) * (C * 9) + n * 9 + (k >> 5)];
    };
    float ra[NA], rb[NB];
    auto load = [&](int k0) {
#pragma unroll
        for (int i = 0; i < NA; ++i) {
            int mm, kk; a_at(i, mm, kk);
            const int k = k0 + kk, m = m0 + mm;
            ra[i] = (k < ke && m < M) ? a_val(m, k) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < NB; ++i) {
            int nn, kk; b_at(i, nn, kk);
            const int k = k0 + kk, n = n0 + nn;
            rb[i] = (k < ke && n < N) ? b_val(k, n) : 0.f;
        }
    };
    float d[BN / 2], acc[BN / 2];                          // d: this k tile's sum (tensor core), acc: the chunk's sum (FADD, round to nearest)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { d[i] = 0.f; acc[i] = 0.f; }
    const uint32_t sa = b200::smem_u32(&sA[0][0][0]), sb = b200::smem_u32(&sB[0][0][0]);
    load(kb);
    for (int k0 = kb; k0 < ke; k0 += TG_BK) {
        __syncthreads();                                   // the previous tile's wgmmas are complete (every thread waited on them)
#pragma unroll
        for (int i = 0; i < NA; ++i) { int mm, kk; a_at(i, mm, kk); sA[kk >> 2][mm][kk & 3] = tf32_rna(ra[i]); }
#pragma unroll
        for (int i = 0; i < NB; ++i) { int nn, kk; b_at(i, nn, kk); sB[kk >> 2][nn][kk & 3] = tf32_rna(rb[i]); }
        b200::fence_async_smem();
        __syncthreads();
        b200::wgmma_fence();
#pragma unroll
        for (int s = 0; s < TG_BK / 8; ++s)
            wgmma_tf32(d, b200::gmma_desc(sa + s * 2 * TG_BM * 16, TG_BM * 16, 128), b200::gmma_desc(sb + s * 2 * BN * 16, BN * 16, 128), s ? 1u : 0u);
        b200::wgmma_commit();
        if (k0 + TG_BK < ke) load(k0 + TG_BK);            // next tile's global loads overlap this tile's MMAs
        b200::wgmma_wait<0>();
        b200::fence_regs(d);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += d[i];
    }
    const int w = tid >> 5, lane = tid & 31, qd = lane & 3, rl = lane >> 2;
    double *Cp = Cdirect ? nullptr : Cpart + (size_t)blockIdx.z * M * N;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = m0 + 16 * w + 8 * h + rl, n = n0 + 8 * j + 2 * qd + e;
                if (m >= M || n >= N) continue;
                const size_t o = ct ? (size_t)n * M + m : (size_t)m * N + n;
                const float a = acc[4 * j + 2 * h + e];
                if (Cdirect) {                             // one k range: bias / ReLU / mask here (no partial-sum buffer)
                    float v = a;
                    if (bias) v = v + bias[n];
                    if (relu) v = fmaxf(v, 0.f);
                    if (mask) v = mask[o] > 0.f ? v : 0.f;
                    Cdirect[o] = v;
                } else {
                    Cp[o] = (double)a;
                }
            }
}

// out[i] = float(sum_z part[z][i] (+ bias[i % N] when bias)), optional ReLU; also used to finish single-split GEMMs.  T = double: the
// unrounded fp64 sum (a data-parallel gradient slice, b200_trainer_grad_rows_dev; no bias / ReLU there)
template <typename T>
__global__ void k_finish(const double *__restrict__ part, int splits, size_t MN, int N, const float *__restrict__ bias, int relu, T *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < MN; i += (size_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int z = 0; z < splits; ++z) s += part[(size_t)z * MN + i];
        if (sizeof(T) == sizeof(double)) { out[i] = (T)s; continue; }
        float v = (float)s;
        if (bias) v = v + bias[i % N];
        if (relu) v = fmaxf(v, 0.f);
        out[i] = v;
    }
}

// column sums: out[n] = T(sum_m X[m][n]) in fp64, one CTA per 32 columns, fixed order (rows strided over 8 warps, then a tree)
template <typename T>
__global__ void __launch_bounds__(256) k_colsum(const float *__restrict__ X, int M, int N, T *__restrict__ out) {
    __shared__ double s[8][32];
    const int n = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
    double a = 0.0;
    if (n < N) for (int m = w; m < M; m += 8) a += (double)X[(size_t)m * N + n];
    s[w][threadIdx.x & 31] = a;
    __syncthreads();
    if (w == 0 && n < N) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += s[i][threadIdx.x & 31];
        out[n] = (T)t;
    }
}

// ------------------------------------------------------------------------------------------------ layout kernels
__global__ void k_states_to_float(const int8_t *s, size_t n, float *x) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] = (float)s[i];
}
// gather a batch from 212-byte replay rows {int8 state[200], f32 value, f32 variance, f32 visit} (include/b200_tetris_mcts.h)
__global__ void k_gather_rows(const uint8_t *rows, const int32_t *idx, int n, float wscale, float *x, float *value, float *variance, float *weight) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n * 203; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / 203), c = (int)(i % 203);
        const uint8_t *r = rows + (size_t)idx[b] * 212;
        if (c < 200) x[(size_t)b * 200 + c] = (float)(int8_t)r[c];
        else {
            float f;
            memcpy(&f, r + 200 + 4 * (c - 200), 4);
            if (c == 200) value[b] = f; else if (c == 201) variance[b] = f; else weight[b] = f * wscale;
        }
    }
}
// im2col of a [B][H][W][C] (NHWC) activation for a valid 3x3 convolution: col[(b, y, x)][ci*9 + ky*3 + kx]
__global__ void k_im2col(const float *__restrict__ act, int B, int H, int W, int C, float *__restrict__ col) {
    const int OH = H - 2, OW = W - 2, K = C * 9;
    const size_t total = (size_t)B * OH * OW * K;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % K);
        const size_t m = i / K;
        const int x = (int)(m % OW), y = (int)((m / OW) % OH), b = (int)(m / ((size_t)OW * OH));
        const int ci = k / 9, tap = k % 9, ky = tap / 3, kx = tap % 3;
        col[i] = act[(((size_t)b * H + y + ky) * W + x + kx) * C + ci];
    }
}
// the adjoint: dact[b][yy][xx][ci] = sum over the <= 9 (output pixel, tap) pairs that read it, ascending tap order; masked by act > 0 (ReLU)
__global__ void k_col2im_relu(const float *__restrict__ dcol, const float *__restrict__ act, int B, int H, int W, int C, float *__restrict__ dact) {
    const int OH = H - 2, OW = W - 2, K = C * 9;
    const size_t total = (size_t)B * H * W * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ci = (int)(i % C);
        const size_t p = i / C;
        const int xx = (int)(p % W), yy = (int)((p / W) % H), b = (int)(p / ((size_t)W * H));
        double s = 0.0;
        for (int ky = 0; ky < 3; ++ky)
            for (int kx = 0; kx < 3; ++kx) {
                const int y = yy - ky, x = xx - kx;
                if (y >= 0 && y < OH && x >= 0 && x < OW) s += (double)dcol[(((size_t)b * OH + y) * OW + x) * K + ci * 9 + ky * 3 + kx];
            }
        dact[i] = act[i] > 0.f ? (float)s : 0.f;
    }
}
// conv3 output [B*56][32] (NHWC rows) <-> the flatten order of nn.Flatten on NCHW: flat[b][c*56 + p]
__global__ void k_nhwc_to_flat(const float *__restrict__ a, int B, float *__restrict__ flat) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * 1792; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / 1792), k = (int)(i % 1792), c = k / 56, p = k % 56;
        flat[i] = a[((size_t)b * 56 + p) * 32 + c];
    }
}
__global__ void k_flat_to_nhwc_relu(const float *__restrict__ dflat, const float *__restrict__ flat, int B, float *__restrict__ d) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * 1792; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / 1792), k = (int)(i % 1792), c = k / 56, p = k % 56;
        d[((size_t)b * 56 + p) * 32 + c] = flat[i] > 0.f ? dflat[i] : 0.f;
    }
}

// ------------------------------------------------------------------------------------------------ head: fc_out, sigmoid, bounds, loss
// One thread per sample of B (a slice of a batch of Bg rows; Bg = B but in b200_trainer_grad_rows_dev): z = h . Wo^T + bo (fp64 accumulate), s = sigmoid(z), pred = s * ub + lb (model_vv.py:48-52), GaussianLL
// (model_vv.py:94-101) with the target variance clamped at 0.1 (:140), weight applied when `weighted` (:145-149); and the gradient of
// mean(w * logl) with respect to z (the two pre-sigmoid outputs).
__global__ void k_head(const float *__restrict__ h, const float *__restrict__ Wo, const float *__restrict__ bo, const float *__restrict__ ub,
                       const float *__restrict__ lb, const float *__restrict__ value, const float *__restrict__ variance, const float *__restrict__ weight,
                       int B, int Bg, int weighted, float *__restrict__ pred, float *__restrict__ lossv, float *__restrict__ dz) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double z0 = 0.0, z1 = 0.0;
    for (int k = 0; k < 256; ++k) { const double hv = (double)h[(size_t)b * 256 + k]; z0 = fma(hv, (double)Wo[k], z0); z1 = fma(hv, (double)Wo[256 + k], z1); }
    const float x0 = (float)z0 + bo[0], x1 = (float)z1 + bo[1];
    const float s0 = 1.f / (1.f + expf(-x0)), s1 = 1.f / (1.f + expf(-x1));
    const float mp = __fadd_rn(__fmul_rn(s0, ub[0]), lb[0]), vp = __fadd_rn(__fmul_rn(s1, ub[1]), lb[1]);
    pred[2 * b] = mp; pred[2 * b + 1] = vp;
    if (!lossv) return;
    const float var = fmaxf(variance[b], 0.1f), mean = value[b];
    const float diff = mean - mp;
    const float t2 = (diff * diff + var) / vp;
    float l = logf(vp) + t2;
    l = l + (-1.f) * logf(var);
    l = l + (-1.f);
    const float w = weighted ? weight[b] : 1.f;
    lossv[b] = w * l;
    if (!dz) return;
    const float gl = w / (float)Bg;                                 // d mean(w * logl) / d logl_b over the whole batch of Bg rows
    const float dvp = gl * (1.f / vp - t2 / vp);                    // d/d var_pred
    const float dmp = gl * (-2.f * diff / vp);                      // d/d mean_pred
    dz[2 * b] = dmp * ub[0] * (s0 * (1.f - s0));
    dz[2 * b + 1] = dvp * ub[1] * (s1 * (1.f - s1));
}
// torch.std_mean(x, unbiased=False): one CTA, fp64
__global__ void __launch_bounds__(256) k_std_mean(const float *__restrict__ x, int n, double *out2) {
    __shared__ double s[256];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) a += (double)x[i];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    const double mean = s[0] / n;
    __syncthreads();
    a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) { const double d = (double)x[i] - mean; a += d * d; }
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) { out2[0] = mean; out2[1] = sqrt(s[0] / n); }
}
// the same two passes, written as the moments {n, mean, M2 = sum (x - mean)^2} of a batch slice (k_loss_combine joins the slices)
__global__ void __launch_bounds__(256) k_moments(const float *__restrict__ x, int n, double *out3) {
    __shared__ double s[256];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) a += (double)x[i];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    const double mean = s[0] / n;
    __syncthreads();
    a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) { const double d = (double)x[i] - mean; a += d * d; }
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) { out3[0] = (double)n; out3[1] = mean; out3[2] = s[0]; }
}
// dh[b][k] = (dz[b][0] * Wo[0][k] + dz[b][1] * Wo[1][k]) masked by h > 0
__global__ void k_dh(const float *__restrict__ dz, const float *__restrict__ Wo, const float *__restrict__ h, int B, float *__restrict__ dh) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B * 256; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i >> 8), k = (int)(i & 255);
        const double v = fma((double)dz[2 * b], (double)Wo[k], (double)dz[2 * b + 1] * (double)Wo[256 + k]);
        dh[i] = h[i] > 0.f ? (float)v : 0.f;
    }
}
// sum of squares per parameter tensor (gradient norm, model/model.py:85-93), fp64, one CTA per tensor
__global__ void __launch_bounds__(256) k_sumsq(const float *__restrict__ g, const int *__restrict__ off, double *__restrict__ out) {
    __shared__ double s[256];
    const int lo = off[blockIdx.x], hi = off[blockIdx.x + 1];
    double a = 0.0;
    for (int i = lo + threadIdx.x; i < hi; i += 256) a += (double)g[i] * (double)g[i];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) out[blockIdx.x] = s[0];
}
__global__ void k_scale(float *g, int n, float c) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) g[i] *= c;
}

// ------------------------------------------------------------------------------------------------ Yogi (model/yogi.py:39-90), elementwise in fp32
struct YogiConst { float beta1, one_minus_beta1, neg_one_minus_beta2, wd, eps, sqrt_bc2, step_size; int first; };
__global__ void k_yogi(float *__restrict__ p, const float *__restrict__ grad, float *__restrict__ m, float *__restrict__ v, int n, YogiConst c) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float g = grad[i];
        float mi = m[i], vi = v[i];
        if (c.first) { mi = 0.f; vi = __fmul_rn(g, g); }                                    // yogi.py:58-61 (exp_avg_sq from the RAW gradient)
        if (c.wd != 0.f) g = __fadd_rn(g, __fmul_rn(c.wd, p[i]));                           // :70-71 grad.add(weight_decay, p.data)
        mi = __fadd_rn(__fmul_rn(mi, c.beta1), __fmul_rn(c.one_minus_beta1, g));            // :74 exp_avg.mul_(beta1).add_(1 - beta1, grad)
        const float gs = __fmul_rn(g, g);                                                   // :76
        const float d = __fsub_rn(vi, gs);
        const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);                            // torch.sign
        vi = __fadd_rn(vi, __fmul_rn(c.neg_one_minus_beta2, __fmul_rn(sg, gs)));            // :78-82 addcmul_
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), c.sqrt_bc2), c.eps);        // :84-86
        p[i] = __fadd_rn(p[i], __fmul_rn(-c.step_size, __fdiv_rn(mi, denom)));              // :87-88 addcdiv_
        m[i] = mi; v[i] = vi;
    }
}

// ------------------------------------------------------------------------------------------------ device-side training loop (b200_trainer_train_rows_dev)
// batch indices: idx[i] = splitmix64(splitmix64(splitmix64(seed) + iteration) + i) mod n_rows (include/b200_tetris_mcts.h)
__host__ __device__ inline uint64_t splitmix64(uint64_t x) {
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
// rows [first, first + n) of the batch: idx[i] is global row first + i
__global__ void k_sample_idx(int32_t *idx, int n, int n_rows, uint64_t seed, uint64_t iteration, int first) {
    const uint64_t base = splitmix64(splitmix64(seed) + iteration);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        idx[i] = (int32_t)(splitmix64(base + (uint64_t)first + (uint64_t)i) % (uint64_t)n_rows);
}
__global__ void k_seq_idx(int32_t *idx, int n, int first) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idx[i] = first + i;
}
// step_common's host arithmetic on the device, operation for operation (no contraction into FMAs): gn = sqrt(sum_i sqrt(ss_i)^2) in tensor order,
// coef = clip / (gn + 1e-6); out_gn <- gn; coef_out <- (float)coef when clipping applies (coef < 1), else -1 (k_scale_dev then leaves the gradient)
__global__ void k_grad_norm(const double *__restrict__ ss, double grad_clip, double *__restrict__ out_gn, float *__restrict__ coef_out) {
    double tot = 0.0;
    for (int i = 0; i < N_TENSORS; ++i) { const double nrm = __dsqrt_rn(ss[i]); tot = __dadd_rn(tot, __dmul_rn(nrm, nrm)); }
    const double gn = __dsqrt_rn(tot);
    *out_gn = gn;
    float c = -1.f;
    if (grad_clip > 0.0) { const double coef = __ddiv_rn(grad_clip, __dadd_rn(gn, 1e-6)); if (coef < 1.0) c = (float)coef; }
    *coef_out = c;
}
__global__ void k_scale_dev(float *g, int n, const float *__restrict__ coef) {
    const float c = *coef;
    if (c < 0.f) return;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) g[i] *= c;
}
// sum of the batch weights in fp64 (the chunk size Model.compute_loss weighs a weighted chunk with, model/model.py:69-70), one CTA, fixed order
__global__ void __launch_bounds__(256) k_sum(const float *__restrict__ x, int n, double *out) {
    __shared__ double s[256];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) a += (double)x[i];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) *out = s[0];
}
// max(value), max(variance), sum(visit) (fp64) of rows [0, n): per-CTA partials over a fixed grid-stride, then one CTA adds them in CTA order
constexpr int STATS_CTAS = 132;
__global__ void __launch_bounds__(256) k_rows_stats_part(const uint8_t *__restrict__ rows, int n, float *__restrict__ pmax, double *__restrict__ psum) {
    __shared__ float s_v[256], s_var[256];
    __shared__ double s_w[256];
    float mv = -INFINITY, mvar = -INFINITY;
    double w = 0.0;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += STATS_CTAS * 256) {
        float f[3];
        memcpy(f, rows + (size_t)i * 212 + 200, 12);
        mv = fmaxf(mv, f[0]); mvar = fmaxf(mvar, f[1]); w += (double)f[2];
    }
    s_v[threadIdx.x] = mv; s_var[threadIdx.x] = mvar; s_w[threadIdx.x] = w;
    __syncthreads();
    for (int d = 128; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            s_v[threadIdx.x] = fmaxf(s_v[threadIdx.x], s_v[threadIdx.x + d]); s_var[threadIdx.x] = fmaxf(s_var[threadIdx.x], s_var[threadIdx.x + d]);
            s_w[threadIdx.x] += s_w[threadIdx.x + d];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) { pmax[2 * blockIdx.x] = s_v[0]; pmax[2 * blockIdx.x + 1] = s_var[0]; psum[blockIdx.x] = s_w[0]; }
}
__global__ void k_rows_stats_final(const float *__restrict__ pmax, const double *__restrict__ psum, float *__restrict__ out_max, double *__restrict__ out_sum) {
    float mv = -INFINITY, mvar = -INFINITY;
    double w = 0.0;
    for (int b = 0; b < STATS_CTAS; ++b) { mv = fmaxf(mv, pmax[2 * b]); mvar = fmaxf(mvar, pmax[2 * b + 1]); w += psum[b]; }
    out_max[0] = mv; out_max[1] = mvar; *out_sum = w;
}

// ------------------------------------------------------------------------------------------------ data-parallel step (b200_trainer_apply_grads_dev)
// parts: n_parts vectors of `stride` doubles (one per rank, ascending rank), each the unrounded fp64 gradient of a batch slice followed by
// that slice's loss moments.  g[i] = (float)(((p0 + p1) + p2) + ...): one left-to-right fp64 sum in part order, rounded once.
__global__ void k_grad_reduce(const double *__restrict__ parts, int n_parts, size_t stride, int n, float *__restrict__ g) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        double s = parts[i];
        for (int r = 1; r < n_parts; ++r) s += parts[(size_t)r * stride + i];
        g[i] = (float)s;
    }
}
// the slices' {count, mean, M2} joined in part order (Chan et al.'s pairwise update) -> lg[0] = mean, lg[1] = population std
__global__ void k_loss_combine(const double *__restrict__ mom, int n_parts, size_t stride, double *__restrict__ lg) {
    double n = mom[0], mean = mom[1], m2 = mom[2];
    for (int r = 1; r < n_parts; ++r) {
        const double *q = mom + (size_t)r * stride;
        const double nb = q[0], d = q[1] - mean, nn = n + nb;
        mean = mean + d * nb / nn;
        m2 = m2 + q[2] + d * d * n * nb / nn;
        n = nn;
    }
    lg[0] = mean; lg[1] = sqrt(m2 / n);
}

inline int nblk(size_t n, int t = 256) { size_t b = (n + t - 1) / t; return (int)(b < 1 ? 1 : (b > 132 * 16 ? 132 * 16 : b)); }

}  // namespace

struct b200_trainer {
    int device = 0, max_batch = 0, kind = B200_TRAIN_FP64;
    cudaStream_t stream = nullptr; bool own_stream = true;              // own_stream false: the caller's (b200_trainer_set_stream), never destroyed here
    std::vector<void *> allocs;
    float *w = nullptr, *grad = nullptr, *m = nullptr, *v = nullptr;     // [N_ALL] / [N_TRAIN]
    int *d_toff = nullptr; double *d_sumsq = nullptr, *d_lossstat = nullptr;
    long long step = 0; bool have_state = false;
    double lr = 1e-3, beta1 = 0.9, beta2 = 0.999, eps = 1e-3, wd = 1e-3;  // Yogi(lr=1e-3, eps=1e-3, weight_decay=1e-3), model_vv.py:132; betas yogi.py:13
    // batch buffers
    int8_t *d_states = nullptr; int32_t *d_idx = nullptr;
    float *x0, *value, *variance, *weight;
    float *col1, *a1, *col2, *a2, *col3, *a3, *flat, *h, *pred, *lossv, *dz;
    float *dh, *dflat, *dc3, *dcol3, *da2, *dcol2, *da1;
    double *part; size_t part_elems = 0;                                // split-k / chunk partial sums (fp64)
    // b200_trainer_train_rows_dev / _loss_rows_dev / b200_rows_stats_dev
    float *d_coef = nullptr, *d_pmax = nullptr, *d_max2 = nullptr; double *d_psum = nullptr, *d_dsum = nullptr;
    double *d_log = nullptr; size_t log_cap = 0;                         // [slots][3] step log, grown on demand (not in allocs)
};

namespace {

template <typename T> int talloc(b200_trainer *t, T **p, size_t n) {
    void *q = nullptr;
    if (cudaMalloc(&q, (n ? n : 1) * sizeof(T)) != cudaSuccess) return tfail(B200_ERR_CUDA, "cudaMalloc failed (trainer, " + std::to_string(n * sizeof(T)) + " B)");
    t->allocs.push_back(q);
    *p = (T *)q;
    return 0;
}

// C = op(A) op(B) with fp64 accumulation, optional bias / ReLU; split-k for long reductions (fixed order).  out64 (no bias / ReLU): C is not
// written; out64 gets the fp64 values C would be rounded from (the accumulator itself for one k range, k_finish's sum for several).
template <bool TA, bool TB>
int gemm(b200_trainer *t, const float *A, const float *B, float *C, int M, int N, int K, const float *bias, int relu, double *out64 = nullptr) {
    int splits = 1;
    const int tiles = ((M + 63) / 64) * ((N + 63) / 64);
    if (K >= 4096 && tiles < 132 * 2) { splits = (132 * 4 + tiles - 1) / tiles; if (splits > (K + 511) / 512) splits = (K + 511) / 512; }
    int kps = ((K + splits - 1) / splits + 15) / 16 * 16;
    splits = (K + kps - 1) / kps;
    dim3 grid((N + 63) / 64, (M + 63) / 64, splits);
    if (splits == 1) {
        if (out64) k_gemm<TA, TB><<<grid, 256, 0, t->stream>>>(A, B, out64, M, N, K, kps, nullptr, nullptr, 0);
        else k_gemm<TA, TB><<<grid, 256, 0, t->stream>>>(A, B, nullptr, M, N, K, kps, C, bias, relu);
        return 0;
    }
    if ((size_t)splits * M * N > t->part_elems) return tfail(B200_ERR_BAD_ARG, "trainer: partial-sum buffer too small");
    k_gemm<TA, TB><<<grid, 256, 0, t->stream>>>(A, B, t->part, M, N, K, kps, nullptr, nullptr, 0);
    if (out64) k_finish<double><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, N, nullptr, 0, out64);
    else k_finish<float><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, N, bias, relu, C);
    return 0;
}

// k ranges of a tc GEMM, from the shapes alone: chunks of <= TG_KCHUNK (the fp32 chain cap), and when the output has too few tiles to fill
// the GPU (< 2 x 132 CTAs), more ranges of >= 256 k.  In that second case splits <= ceil(264 / tiles) and M*N <= tiles * 64 * 64, so the
// partials take <= (264 + tiles) * 4096 < 528 * 4096 doubles (tc_part_elems).
inline int tc_k_per_split(int M, int N, int K, int BN) {
    const int tiles = ((M + TG_BM - 1) / TG_BM) * ((N + BN - 1) / BN);
    int splits = (K + TG_KCHUNK - 1) / TG_KCHUNK;
    if (K >= 512 && tiles * splits < 132 * 2) splits = std::max(splits, std::min((132 * 2 + tiles - 1) / tiles, K / 256));
    return ((K + splits - 1) / splits + TG_BK - 1) / TG_BK * TG_BK;
}

// C = op(A) op(B) on tensor cores (k_gemm_tc), optional bias / ReLU; ct: C stored transposed; out64 as in gemm (the fp32 accumulator of one
// k range is exact in fp64)
template <bool TA, bool TB, int BN>
int gemm_tc(b200_trainer *t, const float *A, const float *B, float *C, int M, int N, int K, const float *bias, int relu, int ct = 0,
            double *out64 = nullptr) {
    const int kps = tc_k_per_split(M, N, K, BN), splits = (K + kps - 1) / kps;
    dim3 grid((N + BN - 1) / BN, (M + TG_BM - 1) / TG_BM, splits);
    if (splits == 1) {
        if (out64) k_gemm_tc<TA, TB, BN><<<grid, 128, 0, t->stream>>>(A, B, out64, M, N, K, kps, nullptr, nullptr, 0, ct);
        else k_gemm_tc<TA, TB, BN><<<grid, 128, 0, t->stream>>>(A, B, nullptr, M, N, K, kps, C, bias, relu, ct);
        return 0;
    }
    if ((size_t)splits * M * N > t->part_elems) return tfail(B200_ERR_BAD_ARG, "trainer: partial-sum buffer too small");
    k_gemm_tc<TA, TB, BN><<<grid, 128, 0, t->stream>>>(A, B, t->part, M, N, K, kps, nullptr, nullptr, 0, ct);
    if (out64) k_finish<double><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, ct ? M : N, nullptr, 0, out64);
    else k_finish<float><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, ct ? M : N, bias, relu, C);
    return 0;
}

// gemm_tc's launch for k_gemm_tf32 (same k ranges); mask: the ReLU mask of an input gradient, which needs a single k range
template <int AOP, int BOP, int BN, int H = 0, int W = 0, int C = 0>
int gemm_tf32(b200_trainer *t, const float *A, const float *B, float *Cm, int M, int N, int K, const float *bias, int relu, int ct = 0,
              double *out64 = nullptr, const float *mask = nullptr) {
    const int kps = tc_k_per_split(M, N, K, BN), splits = (K + kps - 1) / kps;
    dim3 grid((N + BN - 1) / BN, (M + TG_BM - 1) / TG_BM, splits);
    if (splits == 1) {
        if (out64) k_gemm_tf32<AOP, BOP, BN, H, W, C><<<grid, 128, 0, t->stream>>>(A, B, out64, M, N, K, kps, nullptr, nullptr, 0, ct, nullptr);
        else k_gemm_tf32<AOP, BOP, BN, H, W, C><<<grid, 128, 0, t->stream>>>(A, B, nullptr, M, N, K, kps, Cm, bias, relu, ct, mask);
        return 0;
    }
    if (mask) return tfail(B200_ERR_BAD_ARG, "trainer: a masked product needs one k range");
    if ((size_t)splits * M * N > t->part_elems) return tfail(B200_ERR_BAD_ARG, "trainer: partial-sum buffer too small");
    k_gemm_tf32<AOP, BOP, BN, H, W, C><<<grid, 128, 0, t->stream>>>(A, B, t->part, M, N, K, kps, nullptr, nullptr, 0, ct, nullptr);
    if (out64) k_finish<double><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, ct ? M : N, nullptr, 0, out64);
    else k_finish<float><<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, ct ? M : N, bias, relu, Cm);
    return 0;
}

// the partial-sum buffer of the tc kind at max_batch: the conv / fc1 weight gradients in TG_KCHUNK chunks, or the small-grid bound above
size_t tc_part_elems(int max_batch) {
    const size_t B = (size_t)max_batch;
    auto chunks = [](size_t K) { return (K + TG_KCHUNK - 1) / TG_KCHUNK; };
    size_t n = (size_t)528 * 4096;
    n = std::max(n, chunks(B) * 256 * 1792);                 // fc1
    n = std::max(n, chunks(B * 144) * 9 * 32);               // conv1
    n = std::max(n, chunks(B * 96) * 288 * 32);              // conv2 (conv3 reduces over fewer pixels)
    return n;
}

// C = op(A) op(B) (+ bias, ReLU) in the trainer's kind; BN is the tc kernel's tile width for this shape
template <bool TA, bool TB, int BN>
int mm(b200_trainer *t, const float *A, const float *B, float *C, int M, int N, int K, const float *bias, int relu, double *out64 = nullptr) {
    if (t->kind == B200_TRAIN_TC) return gemm_tc<TA, TB, BN>(t, A, B, C, M, N, K, bias, relu, 0, out64);
    if (t->kind == B200_TRAIN_TF32) return gemm_tf32<TA ? OP_T : OP_N, TB ? OP_T : OP_N, BN>(t, A, B, C, M, N, K, bias, relu, 0, out64);
    return gemm<TA, TB>(t, A, B, C, M, N, K, bias, relu, out64);
}
// The tf32 kind's convolution of act [B][H][W][C] -> out [B][H-2][W-2][32] (+ bias, ReLU), its weight gradient dW[32][C*9] (computed as
// dW^T = col^T dout, stored transposed, like the tc kind's) and, when din, its input gradient din [B][H][W][C] masked by act > 0, each one
// k_gemm_tf32 reading act / dout directly
template <int H, int W, int C>
int conv_fwd_tf32(b200_trainer *t, const float *act, const float *Wt, const float *bias, float *out, int B) {
    return gemm_tf32<OP_CONV, OP_T, 32, H, W, C>(t, act, Wt, out, B * (H - 2) * (W - 2), 32, C * 9, bias, 1);
}
template <int H, int W, int C>
int conv_back_tf32(b200_trainer *t, const float *act, const float *dout, const float *Wt, float *dW, double *dW64, float *din, int B) {
    int rc = gemm_tf32<OP_CONV_T, OP_N, 32, H, W, C>(t, act, dout, dW, C * 9, 32, B * (H - 2) * (W - 2), nullptr, 0, 1, dW64);
    if constexpr (C == 32) {                           // OP_DGRAD's k order takes 32 channels per tap (conv1 needs no input gradient)
        if (din) rc |= gemm_tf32<OP_DGRAD, OP_DGRAD_W, 32, H, W, C>(t, dout, Wt, din, B * H * W, 32, 9 * 32, nullptr, 0, 0, nullptr, act);
    }
    return rc;
}
// conv weight gradient dW[32][Kc] = dout^T [32 x P] . col [P x Kc]; the tc kind computes dW^T = col^T dout (32 output columns) and stores
// it transposed
int conv_wgrad(b200_trainer *t, const float *dout, const float *col, float *dW, int Kc, int P, double *out64) {
    if (t->kind == B200_TRAIN_TC) return gemm_tc<true, false, 32>(t, col, dout, dW, Kc, 32, P, nullptr, 0, 1, out64);
    return gemm<true, false>(t, dout, col, dW, 32, Kc, P, nullptr, 0, out64);
}
// bias gradients: column sums of X [M][N], rounded to out or (g64) unrounded
void colsum(b200_trainer *t, const float *X, int M, int N, float *out, double *out64) {
    if (out64) k_colsum<double><<<(N + 31) / 32, 256, 0, t->stream>>>(X, M, N, out64);
    else k_colsum<float><<<(N + 31) / 32, 256, 0, t->stream>>>(X, M, N, out);
}

int forward(b200_trainer *t, int B) {
    float *W = t->w;
    int rc = 0;
    if (t->kind == B200_TRAIN_TF32) {                                                                // implicit im2col
        rc |= conv_fwd_tf32<20, 10, 1>(t, t->x0, W + O_C1W, W + O_C1B, t->a1, B);
        rc |= conv_fwd_tf32<18, 8, 32>(t, t->a1, W + O_C2W, W + O_C2B, t->a2, B);
        rc |= conv_fwd_tf32<16, 6, 32>(t, t->a2, W + O_C3W, W + O_C3B, t->a3, B);
        k_nhwc_to_flat<<<nblk((size_t)B * 1792), 256, 0, t->stream>>>(t->a3, B, t->flat);
        return rc | mm<false, true, 64>(t, t->flat, W + O_F1W, t->h, B, 256, 1792, W + O_F1B, 1);
    }
    k_im2col<<<nblk((size_t)B * 144 * 9), 256, 0, t->stream>>>(t->x0, B, 20, 10, 1, t->col1);
    rc |= mm<false, true, 32>(t, t->col1, W + O_C1W, t->a1, B * 144, 32, 9, W + O_C1B, 1);        // model_vv.py:32-33
    k_im2col<<<nblk((size_t)B * 96 * 288), 256, 0, t->stream>>>(t->a1, B, 18, 8, 32, t->col2);
    rc |= mm<false, true, 32>(t, t->col2, W + O_C2W, t->a2, B * 96, 32, 288, W + O_C2B, 1);        // :34-35
    k_im2col<<<nblk((size_t)B * 56 * 288), 256, 0, t->stream>>>(t->a2, B, 16, 6, 32, t->col3);
    rc |= mm<false, true, 32>(t, t->col3, W + O_C3W, t->a3, B * 56, 32, 288, W + O_C3B, 1);        // :36-37
    k_nhwc_to_flat<<<nblk((size_t)B * 1792), 256, 0, t->stream>>>(t->a3, B, t->flat);              // :38 nn.Flatten on NCHW
    rc |= mm<false, true, 64>(t, t->flat, W + O_F1W, t->h, B, 256, 1792, W + O_F1B, 1);            // :39-40
    return rc;
}

int upload_batch(b200_trainer *t, const int8_t *states, const float *value, const float *variance, const float *weight, int n) {
    if (!states || !value || !variance || n < 1 || n > t->max_batch) return tfail(B200_ERR_BAD_ARG, "trainer: bad batch (1 <= n <= max_batch)");
    TCK(cudaMemcpyAsync(t->d_states, states, (size_t)n * 200, cudaMemcpyHostToDevice, t->stream));
    TCK(cudaMemcpyAsync(t->value, value, (size_t)n * 4, cudaMemcpyHostToDevice, t->stream));
    TCK(cudaMemcpyAsync(t->variance, variance, (size_t)n * 4, cudaMemcpyHostToDevice, t->stream));
    if (weight) TCK(cudaMemcpyAsync(t->weight, weight, (size_t)n * 4, cudaMemcpyHostToDevice, t->stream));
    k_states_to_float<<<nblk((size_t)n * 200), 256, 0, t->stream>>>(t->d_states, (size_t)n * 200, t->x0);
    return 0;
}

int loss_and_head(b200_trainer *t, int B, int weighted, bool want_grad, double *loss, double *loss_std) {
    float *W = t->w;
    k_head<<<(B + 127) / 128, 128, 0, t->stream>>>(t->h, W + O_FOW, W + O_FOB, W + O_UB, W + O_LB, t->value, t->variance, t->weight, B, B,
                                                   weighted, t->pred, t->lossv, want_grad ? t->dz : nullptr);
    k_std_mean<<<1, 256, 0, t->stream>>>(t->lossv, B, t->d_lossstat);
    double h2[2];
    TCK(cudaMemcpyAsync(h2, t->d_lossstat, 16, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    if (loss) *loss = h2[0];
    if (loss_std) *loss_std = h2[1];
    return 0;
}

// the parameter gradient of the B rows in the batch buffers -> t->grad (fp32), or, g64 != nullptr, g64[0 : N_TRAIN] in fp64: the values the
// fp32 gradient would be rounded from (same kernels, same order; only the last rounding is left out)
int backward(b200_trainer *t, int B, double *g64 = nullptr) {
    float *W = t->w, *G = t->grad;
    auto G64 = [&](int off) { return g64 ? g64 + off : nullptr; };
    int rc = 0;
    // fc_out: dWo[j][k] = sum_b dz[b][j] h[b][k]; dbo[j] = sum_b dz[b][j]  (k_gemm in both kinds: 2 x 256 outputs)
    rc |= gemm<true, false>(t, t->dz, t->h, G + O_FOW, 2, 256, B, nullptr, 0, G64(O_FOW));
    colsum(t, t->dz, B, 2, G + O_FOB, G64(O_FOB));
    k_dh<<<nblk((size_t)B * 256), 256, 0, t->stream>>>(t->dz, W + O_FOW, t->h, B, t->dh);
    // fc1: dW1[n][k] = sum_b dh[b][n] flat[b][k]; db1; dflat = dh . W1
    rc |= mm<true, false, 64>(t, t->dh, t->flat, G + O_F1W, 256, 1792, B, nullptr, 0, G64(O_F1W));
    colsum(t, t->dh, B, 256, G + O_F1B, G64(O_F1B));
    rc |= mm<false, false, 64>(t, t->dh, W + O_F1W, t->dflat, B, 1792, 256, nullptr, 0);
    k_flat_to_nhwc_relu<<<nblk((size_t)B * 1792), 256, 0, t->stream>>>(t->dflat, t->flat, B, t->dc3);   // ReLU after conv3 (act3)
    if (t->kind == B200_TRAIN_TF32) {                  // implicit im2col and input gradients (no col / dcol buffers, no col2im)
        rc |= conv_back_tf32<16, 6, 32>(t, t->a2, t->dc3, W + O_C3W, G + O_C3W, G64(O_C3W), t->da2, B);
        colsum(t, t->dc3, B * 56, 32, G + O_C3B, G64(O_C3B));
        rc |= conv_back_tf32<18, 8, 32>(t, t->a1, t->da2, W + O_C2W, G + O_C2W, G64(O_C2W), t->da1, B);
        colsum(t, t->da2, B * 96, 32, G + O_C2B, G64(O_C2B));
        rc |= conv_back_tf32<20, 10, 1>(t, t->x0, t->da1, W + O_C1W, G + O_C1W, G64(O_C1W), nullptr, B);
        colsum(t, t->da1, B * 144, 32, G + O_C1B, G64(O_C1B));
        return rc;
    }
    // conv3
    rc |= conv_wgrad(t, t->dc3, t->col3, G + O_C3W, 288, B * 56, G64(O_C3W));
    colsum(t, t->dc3, B * 56, 32, G + O_C3B, G64(O_C3B));
    rc |= mm<false, false, 64>(t, t->dc3, W + O_C3W, t->dcol3, B * 56, 288, 32, nullptr, 0);
    k_col2im_relu<<<nblk((size_t)B * 96 * 32), 256, 0, t->stream>>>(t->dcol3, t->a2, B, 16, 6, 32, t->da2);
    // conv2
    rc |= conv_wgrad(t, t->da2, t->col2, G + O_C2W, 288, B * 96, G64(O_C2W));
    colsum(t, t->da2, B * 96, 32, G + O_C2B, G64(O_C2B));
    rc |= mm<false, false, 64>(t, t->da2, W + O_C2W, t->dcol2, B * 96, 288, 32, nullptr, 0);
    k_col2im_relu<<<nblk((size_t)B * 144 * 32), 256, 0, t->stream>>>(t->dcol2, t->a1, B, 18, 8, 32, t->da1);
    // conv1 (no input gradient needed)
    rc |= conv_wgrad(t, t->da1, t->col1, G + O_C1W, 9, B * 144, G64(O_C1W));
    colsum(t, t->da1, B * 144, 32, G + O_C1B, G64(O_C1B));
    return rc;
}

// the step's tail on the device, after t->grad holds the fp32 gradient: gradient norm (lg[2]), clip, Yogi
int finish_step_dev(b200_trainer *t, double grad_clip, double *lg) {
    k_sumsq<<<N_TENSORS, 256, 0, t->stream>>>(t->grad, t->d_toff, t->d_sumsq);
    k_grad_norm<<<1, 1, 0, t->stream>>>(t->d_sumsq, grad_clip, lg + 2, t->d_coef);
    if (grad_clip > 0.0) k_scale_dev<<<nblk(N_TRAIN), 256, 0, t->stream>>>(t->grad, N_TRAIN, t->d_coef);
    // Yogi constants from the step counter alone (step_common)
    const bool first = !t->have_state;
    if (first) { t->step = 0; t->have_state = true; }
    t->step += 1;
    const double bc1 = 1.0 - pow(t->beta1, (double)t->step), bc2 = 1.0 - pow(t->beta2, (double)t->step);
    YogiConst c;
    c.beta1 = (float)t->beta1; c.one_minus_beta1 = (float)(1.0 - t->beta1); c.neg_one_minus_beta2 = (float)(-(1.0 - t->beta2));
    c.wd = (float)t->wd; c.eps = (float)t->eps; c.sqrt_bc2 = (float)sqrt(bc2); c.step_size = (float)(t->lr / bc1); c.first = first ? 1 : 0;
    k_yogi<<<nblk(N_TRAIN), 256, 0, t->stream>>>(t->w, t->grad, t->m, t->v, N_TRAIN, c);
    return 0;
}

// the device step log holds at least `slots` rows of 3; earlier rows are kept
int ensure_log(b200_trainer *t, size_t slots) {
    if (slots * 3 <= t->log_cap) return 0;
    double *nl = nullptr;
    TCK(cudaStreamSynchronize(t->stream));
    TCK(cudaMalloc(&nl, slots * 3 * sizeof(double)));
    if (t->d_log) {
        const cudaError_t e = cudaMemcpy(nl, t->d_log, t->log_cap * sizeof(double), cudaMemcpyDeviceToDevice);
        cudaFree(t->d_log);
        t->d_log = nl; t->log_cap = slots * 3;
        TCK(e);
        return 0;
    }
    t->d_log = nl; t->log_cap = slots * 3;
    return 0;
}

}  // namespace

extern "C" const char *b200_trainer_last_error(void) { return g_terr.c_str(); }

extern "C" int b200_trainer_destroy(b200_trainer *t) {
    if (!t) return B200_OK;
    if (t->stream) cudaStreamSynchronize(t->stream);
    for (void *p : t->allocs) cudaFree(p);
    if (t->d_log) cudaFree(t->d_log);
    if (t->stream && t->own_stream) cudaStreamDestroy(t->stream);
    delete t;
    return B200_OK;
}

extern "C" int b200_trainer_create(int device, const float *weights, int max_batch, b200_trainer **out) {
    return b200_trainer_create_kind(device, weights, max_batch, B200_TRAIN_FP64, out);
}

extern "C" int b200_trainer_create_kind(int device, const float *weights, int max_batch, int kind, b200_trainer **out) {
    if (!weights || !out || max_batch < 1 || max_batch > 65536) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (1 <= max_batch <= 65536)");
    if (kind != B200_TRAIN_FP64 && kind != B200_TRAIN_TC && kind != B200_TRAIN_TF32)
        return tfail(B200_ERR_BAD_ARG, "trainer: unknown kind (B200_TRAIN_FP64, B200_TRAIN_TC or B200_TRAIN_TF32)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return tfail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TCK(cudaSetDevice(device));
    b200_trainer *t = new b200_trainer();
    struct Guard { b200_trainer *t; ~Guard() { if (t) b200_trainer_destroy(t); } } guard{t};
    t->device = device; t->max_batch = max_batch; t->kind = kind;
    TCK(cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking));
    const size_t B = (size_t)max_batch;
    int rc = 0;
    rc |= talloc(t, &t->w, N_ALL); rc |= talloc(t, &t->grad, N_TRAIN); rc |= talloc(t, &t->m, N_TRAIN); rc |= talloc(t, &t->v, N_TRAIN);
    rc |= talloc(t, &t->d_toff, N_TENSORS + 1); rc |= talloc(t, &t->d_sumsq, N_TENSORS); rc |= talloc(t, &t->d_lossstat, 2);
    rc |= talloc(t, &t->d_states, B * 200); rc |= talloc(t, &t->d_idx, B);
    rc |= talloc(t, &t->x0, B * 200); rc |= talloc(t, &t->value, B); rc |= talloc(t, &t->variance, B); rc |= talloc(t, &t->weight, B);
    if (kind != B200_TRAIN_TF32) {                     // the tf32 kind's convolutions read the activations directly (null pointers here)
        rc |= talloc(t, &t->col1, B * 144 * 9); rc |= talloc(t, &t->col2, B * 96 * 288); rc |= talloc(t, &t->col3, B * 56 * 288);
        rc |= talloc(t, &t->dcol3, B * 56 * 288); rc |= talloc(t, &t->dcol2, B * 96 * 288);
    }
    rc |= talloc(t, &t->a1, B * 144 * 32); rc |= talloc(t, &t->a2, B * 96 * 32);
    rc |= talloc(t, &t->a3, B * 56 * 32); rc |= talloc(t, &t->flat, B * 1792); rc |= talloc(t, &t->h, B * 256);
    rc |= talloc(t, &t->pred, B * 2); rc |= talloc(t, &t->lossv, B); rc |= talloc(t, &t->dz, B * 2);
    rc |= talloc(t, &t->dh, B * 256); rc |= talloc(t, &t->dflat, B * 1792); rc |= talloc(t, &t->dc3, B * 56 * 32);
    rc |= talloc(t, &t->da2, B * 96 * 32); rc |= talloc(t, &t->da1, B * 144 * 32);
    // split-k partial sums (fp64): fp64 kind: only the weight-gradient products are split; the largest is fc1 (256 x 1792) with <= 8 k
    // ranges.  tc and tf32 kinds: tc_part_elems (the same k ranges).
    t->part_elems = kind != B200_TRAIN_FP64 ? tc_part_elems(max_batch) : (size_t)8 * 256 * 1792;
    rc |= talloc(t, &t->part, t->part_elems);
    rc |= talloc(t, &t->d_coef, 1); rc |= talloc(t, &t->d_pmax, 2 * STATS_CTAS); rc |= talloc(t, &t->d_psum, STATS_CTAS);
    rc |= talloc(t, &t->d_max2, 2); rc |= talloc(t, &t->d_dsum, 1);
    if (rc) return B200_ERR_CUDA;
    TCK(cudaMemcpyAsync(t->w, weights, N_ALL * sizeof(float), cudaMemcpyHostToDevice, t->stream));
    TCK(cudaMemcpyAsync(t->d_toff, T_OFF, sizeof(T_OFF), cudaMemcpyHostToDevice, t->stream));
    TCK(cudaMemsetAsync(t->m, 0, N_TRAIN * 4, t->stream));
    TCK(cudaMemsetAsync(t->v, 0, N_TRAIN * 4, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    guard.t = nullptr;
    *out = t;
    return B200_OK;
}

extern "C" int b200_trainer_set_hyper(b200_trainer *t, double lr, double beta1, double beta2, double eps, double weight_decay) {
    if (!t || lr <= 0 || eps < 0 || beta1 < 0 || beta1 >= 1 || beta2 < 0 || beta2 >= 1 || weight_decay < 0) return tfail(B200_ERR_BAD_ARG, "trainer: invalid hyper-parameter (yogi.py:14-31)");
    t->lr = lr; t->beta1 = beta1; t->beta2 = beta2; t->eps = eps; t->wd = weight_decay;
    return B200_OK;
}

extern "C" int b200_trainer_set_out_ubound(b200_trainer *t, float ub_value, float ub_variance) {   // model_vv.py:227-231
    if (!t) return tfail(B200_ERR_BAD_ARG, "null trainer");
    TCK(cudaSetDevice(t->device));
    const float ub[2] = {ub_value, ub_variance};
    TCK(cudaMemcpyAsync(t->w + O_UB, ub, 8, cudaMemcpyHostToDevice, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

extern "C" int b200_trainer_get_weights(b200_trainer *t, float *weights_out) {
    if (!t || !weights_out) return tfail(B200_ERR_BAD_ARG, "null argument");
    TCK(cudaSetDevice(t->device));
    TCK(cudaMemcpyAsync(weights_out, t->w, N_ALL * sizeof(float), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

extern "C" int b200_trainer_set_weights(b200_trainer *t, const float *weights) {
    if (!t || !weights) return tfail(B200_ERR_BAD_ARG, "null argument");
    TCK(cudaSetDevice(t->device));
    TCK(cudaMemcpyAsync(t->w, weights, N_ALL * sizeof(float), cudaMemcpyHostToDevice, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// optimizer.state_dict() / load_state_dict (model/model.py:143-171): exp_avg, exp_avg_sq over the trainable parameters in state_dict order, step
extern "C" int b200_trainer_get_state(b200_trainer *t, float *exp_avg, float *exp_avg_sq, int64_t *step) {
    if (!t || !exp_avg || !exp_avg_sq || !step) return tfail(B200_ERR_BAD_ARG, "null argument");
    TCK(cudaSetDevice(t->device));
    TCK(cudaMemcpyAsync(exp_avg, t->m, N_TRAIN * 4, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaMemcpyAsync(exp_avg_sq, t->v, N_TRAIN * 4, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    *step = t->have_state ? t->step : -1;
    return B200_OK;
}
extern "C" int b200_trainer_set_state(b200_trainer *t, const float *exp_avg, const float *exp_avg_sq, int64_t step) {
    if (!t) return tfail(B200_ERR_BAD_ARG, "null trainer");
    TCK(cudaSetDevice(t->device));
    if (step < 0 || !exp_avg || !exp_avg_sq) { t->have_state = false; t->step = 0; return B200_OK; }      // Model.reset_optimizer (model/model.py:134-135)
    TCK(cudaMemcpyAsync(t->m, exp_avg, N_TRAIN * 4, cudaMemcpyHostToDevice, t->stream));
    TCK(cudaMemcpyAsync(t->v, exp_avg_sq, N_TRAIN * 4, cudaMemcpyHostToDevice, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    t->have_state = true; t->step = step;
    return B200_OK;
}

extern "C" int b200_trainer_get_grads(b200_trainer *t, float *grads_out) {      // the gradients of the last b200_trainer_step (parity tests)
    if (!t || !grads_out) return tfail(B200_ERR_BAD_ARG, "null argument");
    TCK(cudaSetDevice(t->device));
    TCK(cudaMemcpyAsync(grads_out, t->grad, N_TRAIN * 4, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// test aid: one batch buffer as the last step / loss / step_rows_dev / grad_rows_dev left it, rows [0, n_rows) (a copy, no kernel)
extern "C" int b200_trainer_debug_buffer(b200_trainer *t, const char *which, int n_rows, void *out) {
    if (!t || !which || !out || n_rows < 0 || n_rows > t->max_batch) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (0 <= n_rows <= max_batch)");
    const struct { const char *name; const float *p; size_t row; } bufs[] = {
        {"x0", t->x0, 200}, {"value", t->value, 1}, {"variance", t->variance, 1}, {"weight", t->weight, 1},
        {"col1", t->col1, 144 * 9}, {"a1", t->a1, 144 * 32}, {"col2", t->col2, 96 * 288}, {"a2", t->a2, 96 * 32},
        {"col3", t->col3, 56 * 288}, {"a3", t->a3, 56 * 32}, {"flat", t->flat, 1792}, {"h", t->h, 256}, {"pred", t->pred, 2},
        {"lossv", t->lossv, 1}, {"dz", t->dz, 2}, {"dh", t->dh, 256}, {"dflat", t->dflat, 1792}, {"dc3", t->dc3, 56 * 32},
        {"dcol3", t->dcol3, 56 * 288}, {"da2", t->da2, 96 * 32}, {"dcol2", t->dcol2, 96 * 288}, {"da1", t->da1, 144 * 32}};
    const void *src = nullptr;
    size_t bytes = 0;
    if (!strcmp(which, "d_sumsq")) { src = t->d_sumsq; bytes = N_TENSORS * sizeof(double); }
    for (const auto &b : bufs)
        if (!strcmp(which, b.name)) {
            if (!b.p) return tfail(B200_ERR_BAD_ARG, std::string("trainer: a tf32 trainer has no buffer ") + which + " (implicit im2col)");
            src = b.p; bytes = (size_t)n_rows * b.row * sizeof(float);
        }
    if (!src) return tfail(B200_ERR_BAD_ARG, std::string("trainer: unknown buffer ") + which);
    TCK(cudaSetDevice(t->device));
    if (bytes) TCK(cudaMemcpyAsync(out, src, bytes, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// Model_VV._loss under torch.no_grad (one chunk of Model.compute_loss, model/model.py:52-83); pred_out (may be NULL): [n][2] = (v, var)
extern "C" int b200_trainer_loss(b200_trainer *t, const int8_t *states, const float *value, const float *variance, const float *weight, int n,
                                 int weighted, double *loss, double *loss_std, float *pred_out) {
    if (!t) return tfail(B200_ERR_BAD_ARG, "null trainer");
    if (weighted && !weight) return tfail(B200_ERR_BAD_ARG, "weighted loss needs weights");
    TCK(cudaSetDevice(t->device));
    int rc = upload_batch(t, states, value, variance, weight, n);
    if (rc) return rc;
    rc = forward(t, n);
    if (rc) return rc;
    rc = loss_and_head(t, n, weighted, false, loss, loss_std);
    if (rc) return rc;
    if (pred_out) { TCK(cudaMemcpyAsync(pred_out, t->pred, (size_t)n * 8, cudaMemcpyDeviceToHost, t->stream)); TCK(cudaStreamSynchronize(t->stream)); }
    TCK(cudaGetLastError());
    return B200_OK;
}

static int step_common(b200_trainer *t, int n, int weighted, double grad_clip, double *loss, double *loss_std, double *grad_norm) {
    int rc = forward(t, n);
    if (rc) return rc;
    rc = loss_and_head(t, n, weighted, true, loss, loss_std);
    if (rc) return rc;
    rc = backward(t, n);
    if (rc) return rc;
    // compute_gradient_norm (model/model.py:85-93): (sum_p ||grad_p||_2^2)^(1/2)
    k_sumsq<<<N_TENSORS, 256, 0, t->stream>>>(t->grad, t->d_toff, t->d_sumsq);
    double ss[N_TENSORS];
    TCK(cudaMemcpyAsync(ss, t->d_sumsq, sizeof(ss), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    double tot = 0.0;
    for (int i = 0; i < N_TENSORS; ++i) { const double nrm = sqrt(ss[i]); tot += nrm * nrm; }
    const double gn = sqrt(tot);
    if (grad_norm) *grad_norm = gn;
    if (grad_clip > 0.0) {                                           // torch.nn.utils.clip_grad_norm_ (model/model.py:110-111)
        const double coef = grad_clip / (gn + 1e-6);
        if (coef < 1.0) k_scale<<<nblk(N_TRAIN), 256, 0, t->stream>>>(t->grad, N_TRAIN, (float)coef);
    }
    // Yogi.step (model/yogi.py:39-90)
    const bool first = !t->have_state;
    if (first) { t->step = 0; t->have_state = true; }
    t->step += 1;
    const double bc1 = 1.0 - pow(t->beta1, (double)t->step), bc2 = 1.0 - pow(t->beta2, (double)t->step);
    YogiConst c;
    c.beta1 = (float)t->beta1; c.one_minus_beta1 = (float)(1.0 - t->beta1); c.neg_one_minus_beta2 = (float)(-(1.0 - t->beta2));
    c.wd = (float)t->wd; c.eps = (float)t->eps; c.sqrt_bc2 = (float)sqrt(bc2); c.step_size = (float)(t->lr / bc1); c.first = first ? 1 : 0;
    k_yogi<<<nblk(N_TRAIN), 256, 0, t->stream>>>(t->w, t->grad, t->m, t->v, N_TRAIN, c);
    TCK(cudaGetLastError());
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// Model.train(batch, grad_clip, weighted) (model/model.py:95-119): one optimiser step on a HOST batch
extern "C" int b200_trainer_step(b200_trainer *t, const int8_t *states, const float *value, const float *variance, const float *weight, int n,
                                 int weighted, double grad_clip, double *loss, double *loss_std, double *grad_norm) {
    if (!t) return tfail(B200_ERR_BAD_ARG, "null trainer");
    if (weighted && !weight) return tfail(B200_ERR_BAD_ARG, "weighted loss needs weights");
    TCK(cudaSetDevice(t->device));
    int rc = upload_batch(t, states, value, variance, weight, n);
    if (rc) return rc;
    return step_common(t, n, weighted, grad_clip, loss, loss_std, grad_norm);
}

// The same step on a batch gathered ON THE DEVICE from 212-byte replay rows (b200_replay_drain_dev / the all-gather block): rows_dev[n_rows],
// idx (host) = the batch's row indices (np.random.choice of Model.train_data, model/model.py:207), weight = visit * weight_scale
// (train_data normalises the weights by their mean, model/model.py:186-187).
extern "C" int b200_trainer_step_rows_dev(b200_trainer *t, const void *rows_dev, int n_rows, const int32_t *idx, int n, float weight_scale,
                                          int weighted, double grad_clip, double *loss, double *loss_std, double *grad_norm) {
    if (!t || !rows_dev || !idx || n < 1 || n > t->max_batch || n_rows < 1) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument");
    for (int i = 0; i < n; ++i) if (idx[i] < 0 || idx[i] >= n_rows) return tfail(B200_ERR_BAD_ARG, "trainer: row index out of range");
    TCK(cudaSetDevice(t->device));
    TCK(cudaMemcpyAsync(t->d_idx, idx, (size_t)n * 4, cudaMemcpyHostToDevice, t->stream));
    k_gather_rows<<<nblk((size_t)n * 203), 256, 0, t->stream>>>((const uint8_t *)rows_dev, t->d_idx, n, weight_scale, t->x0, t->value, t->variance, t->weight);
    return step_common(t, n, weighted, grad_clip, loss, loss_std, grad_norm);
}

// Model.train_data's inner loop (model/model.py:205-212) for `iters` steps on device rows, with one host synchronisation at the end: each step
// draws its batch on the device (k_sample_idx: uniform with replacement over rows [0, n_train_rows), iteration number first_iter + it), then
// runs exactly step_common's kernels; the gradient norm and the clip coefficient are computed on the device with step_common's host arithmetic,
// so every step is bit-identical to b200_trainer_step_rows_dev fed the same indices.  log_out (host) gets [iters][3] = {loss, loss_std, grad_norm}.
extern "C" int b200_trainer_train_rows_dev(b200_trainer *t, const void *rows_dev, int n_train_rows, int batch, int iters, uint64_t seed, int64_t first_iter,
                                           float weight_scale, int weighted, double grad_clip, double *log_out) {
    if (!t || !rows_dev || !log_out || batch < 1 || batch > t->max_batch || n_train_rows < 1 || iters < 0 || first_iter < 0)
        return tfail(B200_ERR_BAD_ARG, "trainer: bad argument");
    TCK(cudaSetDevice(t->device));
    if (iters == 0) return B200_OK;
    int rc = ensure_log(t, (size_t)iters);
    if (rc) return rc;
    float *W = t->w;
    for (int it = 0; it < iters; ++it) {
        double *lg = t->d_log + (size_t)it * 3;
        k_sample_idx<<<nblk(batch), 256, 0, t->stream>>>(t->d_idx, batch, n_train_rows, seed, (uint64_t)(first_iter + it), 0);
        k_gather_rows<<<nblk((size_t)batch * 203), 256, 0, t->stream>>>((const uint8_t *)rows_dev, t->d_idx, batch, weight_scale, t->x0, t->value, t->variance, t->weight);
        rc = forward(t, batch);
        if (rc) return rc;
        k_head<<<(batch + 127) / 128, 128, 0, t->stream>>>(t->h, W + O_FOW, W + O_FOB, W + O_UB, W + O_LB, t->value, t->variance, t->weight, batch, batch,
                                                           weighted, t->pred, t->lossv, t->dz);
        k_std_mean<<<1, 256, 0, t->stream>>>(t->lossv, batch, lg);
        rc = backward(t, batch);
        if (rc) return rc;
        finish_step_dev(t, grad_clip, lg);
    }
    TCK(cudaGetLastError());
    TCK(cudaMemcpyAsync(log_out, t->d_log, (size_t)iters * 3 * sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}

// Model_VV._loss under no_grad on device rows [first, first + n) (one chunk of Model.compute_loss, model/model.py:52-83), weight = visit *
// weight_scale; *weight_sum = the fp64 sum of those weights (the chunk's size in a weighted combination)
extern "C" int b200_trainer_loss_rows_dev(b200_trainer *t, const void *rows_dev, int first, int n, float weight_scale, int weighted,
                                          double *loss, double *loss_std, double *weight_sum) {
    if (!t || !rows_dev || first < 0 || n < 1 || n > t->max_batch) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (1 <= n <= max_batch)");
    TCK(cudaSetDevice(t->device));
    k_seq_idx<<<nblk(n), 256, 0, t->stream>>>(t->d_idx, n, first);
    k_gather_rows<<<nblk((size_t)n * 203), 256, 0, t->stream>>>((const uint8_t *)rows_dev, t->d_idx, n, weight_scale, t->x0, t->value, t->variance, t->weight);
    k_sum<<<1, 256, 0, t->stream>>>(t->weight, n, t->d_dsum);
    double wsum = 0.0;
    TCK(cudaMemcpyAsync(&wsum, t->d_dsum, sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    int rc = forward(t, n);
    if (rc) return rc;
    rc = loss_and_head(t, n, weighted, false, loss, loss_std);      // synchronises the stream
    if (rc) return rc;
    TCK(cudaGetLastError());
    if (weight_sum) *weight_sum = wsum;
    return B200_OK;
}

// max(value), max(variance) and the fp64 sum of visits over rows [0, n) (Model_VV.train_data's out_ubound, model_vv.py:227-231, and the mean of
// Model.train_data's weight normalisation, model/model.py:186-187) without copying the rows to the host; fixed reduction order
extern "C" int b200_rows_stats_dev(b200_trainer *t, const void *rows_dev, int n, float *max_value, float *max_variance, double *visit_sum) {
    if (!t || !rows_dev || n < 1 || !max_value || !max_variance || !visit_sum) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument");
    TCK(cudaSetDevice(t->device));
    k_rows_stats_part<<<STATS_CTAS, 256, 0, t->stream>>>((const uint8_t *)rows_dev, n, t->d_pmax, t->d_psum);
    k_rows_stats_final<<<1, 1, 0, t->stream>>>(t->d_pmax, t->d_psum, t->d_max2, t->d_dsum);
    TCK(cudaGetLastError());
    float mx[2]; double sum = 0.0;
    TCK(cudaMemcpyAsync(mx, t->d_max2, sizeof(mx), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaMemcpyAsync(&sum, t->d_dsum, sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    *max_value = mx[0]; *max_variance = mx[1]; *visit_sum = sum;
    return B200_OK;
}

// All later work of the trainer is issued on `cuda_stream` (nullptr: a private non-blocking stream again); the current stream is drained first.
// The caller keeps ownership of its stream and keeps it alive.  Lets a collective be ordered on the trainer's stream without a host wait.
extern "C" int b200_trainer_set_stream(b200_trainer *t, void *cuda_stream) {
    if (!t) return tfail(B200_ERR_BAD_ARG, "null trainer");
    TCK(cudaSetDevice(t->device));
    TCK(cudaStreamSynchronize(t->stream));
    cudaStream_t ns = (cudaStream_t)cuda_stream;
    const bool own = ns == nullptr;
    if (own) TCK(cudaStreamCreateWithFlags(&ns, cudaStreamNonBlocking));
    if (t->own_stream) cudaStreamDestroy(t->stream);
    t->stream = ns; t->own_stream = own;
    return B200_OK;
}

// Data-parallel step, part 1: rows [lo, hi) of the batch train_rows_dev draws for iteration `iter` (global row numbers in k_sample_idx), forward,
// head with the gradient scale of the whole batch (every sample's dz is the single-GPU step's), backward into grad_dev[0 : N_TRAIN] unrounded
// (fp64), then the slice's loss moments {count, mean, M2} of (weight *) logl in grad_dev[N_TRAIN : N_TRAIN + 3].  Asynchronous.
extern "C" int b200_trainer_grad_rows_dev(b200_trainer *t, const void *rows_dev, int n_train_rows, int batch, int lo, int hi, uint64_t seed, int64_t iter,
                                          float weight_scale, int weighted, double *grad_dev) {
    if (!t || !rows_dev || !grad_dev || n_train_rows < 1 || iter < 0 || lo < 0 || lo >= hi || hi > batch || hi - lo > t->max_batch)
        return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (0 <= lo < hi <= batch, hi - lo <= max_batch)");
    TCK(cudaSetDevice(t->device));
    const int n = hi - lo;
    float *W = t->w;
    k_sample_idx<<<nblk(n), 256, 0, t->stream>>>(t->d_idx, n, n_train_rows, seed, (uint64_t)iter, lo);
    k_gather_rows<<<nblk((size_t)n * 203), 256, 0, t->stream>>>((const uint8_t *)rows_dev, t->d_idx, n, weight_scale, t->x0, t->value, t->variance, t->weight);
    int rc = forward(t, n);
    if (rc) return rc;
    k_head<<<(n + 127) / 128, 128, 0, t->stream>>>(t->h, W + O_FOW, W + O_FOB, W + O_UB, W + O_LB, t->value, t->variance, t->weight, n, batch,
                                                   weighted, t->pred, t->lossv, t->dz);
    k_moments<<<1, 256, 0, t->stream>>>(t->lossv, n, grad_dev + N_TRAIN);
    rc = backward(t, n, grad_dev);
    if (rc) return rc;
    TCK(cudaGetLastError());
    return B200_OK;
}

// Data-parallel step, part 2: g = (float)(p0 + p1 + ... ) in part order (k_grad_reduce), the parts' loss moments joined in part order, then
// train_rows_dev's gradient norm / clip / Yogi.  {loss, loss_std, grad_norm} go to device log slot `log_slot` (b200_trainer_read_log).
// Asynchronous.  One part with the whole batch is bit-identical to a train_rows_dev step (its loss up to reassociation).
extern "C" int b200_trainer_apply_grads_dev(b200_trainer *t, const double *parts_dev, int n_parts, double grad_clip, int log_slot) {
    if (!t || !parts_dev || n_parts < 1 || log_slot < 0) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (n_parts >= 1, log_slot >= 0)");
    TCK(cudaSetDevice(t->device));
    int rc = ensure_log(t, (size_t)log_slot + 1);
    if (rc) return rc;
    double *lg = t->d_log + (size_t)log_slot * 3;
    const size_t stride = (size_t)N_TRAIN + 3;
    k_grad_reduce<<<nblk(N_TRAIN), 256, 0, t->stream>>>(parts_dev, n_parts, stride, N_TRAIN, t->grad);
    k_loss_combine<<<1, 1, 0, t->stream>>>(parts_dev + N_TRAIN, n_parts, stride, lg);
    finish_step_dev(t, grad_clip, lg);
    TCK(cudaGetLastError());
    return B200_OK;
}

// synchronises the trainer's stream and copies log slots [0, n) ([n][3] doubles) to the host
extern "C" int b200_trainer_read_log(b200_trainer *t, int n, double *host) {
    if (!t || n < 0 || (n > 0 && !host) || (size_t)n * 3 > t->log_cap) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (n <= log slots written)");
    TCK(cudaSetDevice(t->device));
    if (n > 0) TCK(cudaMemcpyAsync(host, t->d_log, (size_t)n * 3 * sizeof(double), cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    return B200_OK;
}
