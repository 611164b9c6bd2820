// valuenet_simt.cuh — fp32 CUDA-core forward pass of the reference value network (model/model_vv.py:13-52,
// Model_VV.inference :210-217) over the batch of leaf observations queued by k_select_expand.
//
//   k_vn_conv : obs key -> {-1,0,1} board -> conv1+ReLU -> conv2+ReLU -> conv3+ReLU, all activations in shared
//               memory, 4 boards per CTA pass, persistent CTAs (one per SM) that keep the 73 KB of conv weights
//               resident in shared memory.  Output: act3[request][1792] in HBM, K order (y*32 + c)*4 + x.
//   k_vn_fc   : act3 [R,1792] x W1' [1792,256] (+bias, ReLU) -> fc_out (2 dot products) -> sigmoid -> affine,
//               64x256 output tile per CTA so the whole hidden vector of a row stays in the CTA.
// Arithmetic is plain fp32 in a fixed order: fmaf chains, IEEE adds and divisions, a fixed shuffle tree and an explicit
// __fmul_rn / __fadd_rn affine.  So every activation, fc1 accumulator and logit is one fp32 value, bit for bit the
// restatement of tests/f32_net_ref.py from the previous stage, and each output lies within the few fp32 values that expf's
// 2 ulp admit (tests/test_gpu_net_layers.py, which reads every stage back through the DBG instantiations and
// b200_debug_net_acts).  This is the bit-faithful baseline the tensor-core path (valuenet_tc.cuh) is checked against.
#pragma once
#include "search_dev.cuh"

namespace b200 {

struct NetWeights {          // device pointers, layouts prepared by the host (capi.cu: prepare_weights)
    const float *w1;         // [9][32]      tap-major, cout contiguous
    const float *w2, *w3;    // [288][32]    k = ci*9 + dy*3 + dx, cout contiguous
    const float *b1, *b2, *b3;
    const float *wfc1;       // [1792][256]  k' = (y*32 + c)*4 + x  (torch k = c*56 + y*4 + x), n contiguous
    const float *bfc1;       // [256]
    const float *wout;       // [2][256]
    const float *bout, *ub, *lb;   // [2] each
};

constexpr int VN_TB = 4;              // boards per CTA pass
constexpr int VN_THREADS = 256;
constexpr int VN_SMEM_FLOATS = 9216 * 2 + 288 + 96 + VN_TB * 200 + 32 * VN_TB * 18 * 8 + 32 * VN_TB * 16 * 8;
constexpr int VN_SMEM_BYTES = VN_SMEM_FLOATS * 4;

// Test export of the activations that never leave shared memory: with DBG, each board's act1 [32][18][8] and act2 [32][16][6] are
// copied to dbg + ridx * VN_DBG_FLOATS in [c][y][x] order once conv2 has finished (b200_debug_net_acts returns them).  Only k_vn_conv_dbg
// instantiates it.
constexpr int VN_DBG_A1 = 32 * 18 * 8, VN_DBG_FLOATS = VN_DBG_A1 + 32 * 16 * 6;

template <bool DBG>
__device__ __forceinline__ void vn_conv_body(NetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M, float *act3,
                                             float *dbg) {
    extern __shared__ __align__(16) float sm[];
    float *sW2 = sm;                       // 9216
    float *sW3 = sW2 + 9216;               // 9216
    float *sW1 = sW3 + 9216;               // 288
    float *sB = sW1 + 288;                 // 96: b1 | b2 | b3
    float *sIn = sB + 96;                  // TB*200
    float *sA1 = sIn + VN_TB * 200;        // planes L,R: [2][32][TB*18][4]
    float *sA2 = sA1 + 32 * VN_TB * 18 * 8;   // planes L,R: [2][32][TB*16][4]
    const int t = threadIdx.x;
    for (int i = t; i < 9216; i += VN_THREADS) { sW2[i] = W.w2[i]; sW3[i] = W.w3[i]; }
    for (int i = t; i < 288; i += VN_THREADS) sW1[i] = W.w1[i];
    if (t < 32) { sB[t] = W.b1[t]; sB[32 + t] = W.b2[t]; sB[64 + t] = W.b3[t]; }
    const int n_req = *n_req_ptr;
    const int n_tiles = (n_req + VN_TB - 1) / VN_TB;
    constexpr int A1P = 32 * VN_TB * 18 * 4;   // floats per sA1 plane
    constexpr int A2P = 32 * VN_TB * 16 * 4;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        __syncthreads();
        // ---- decode the observation keys into {-1,0,1} (model_vv.py:212 as_tensor(float))
        for (int i = t; i < VN_TB * 200; i += VN_THREADS) {
            int b = i / 200, cell = i % 200, r = cell / 10, c = cell % 10;
            int ridx = tile * VN_TB + b;
            float v = 0.f;
            if (ridx < n_req) {
                uint2 rq = req[ridx];
                const uint32_t *k = keys + ((size_t)rq.x * M + (rq.y & 0x0fffffffu)) * KEY_WORDS;
                v = (float)((k[r >> 1] >> ((r & 1) * 16 + c)) & 1u);
                uint32_t pc = k[10];
                if ((pc & 0xffu) == (uint32_t)cell || ((pc >> 8) & 0xffu) == (uint32_t)cell ||
                    ((pc >> 16) & 0xffu) == (uint32_t)cell || (pc >> 24) == (uint32_t)cell) v = -1.f;
            }
            sIn[i] = v;
        }
        __syncthreads();
        // ---- conv1 (1->32, 3x3 valid, 20x10 -> 18x8) + ReLU
        for (int task = t; task < VN_TB * 18 * 8 * 4; task += VN_THREADS) {
            int cg = task & 3, pos = task >> 2;
            int x = pos & 7, yb = pos >> 3;            // yb = b*18 + y
            int b = yb / 18, y = yb % 18;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = sB[cg * 8 + j];
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    float in = sIn[b * 200 + (y + dy) * 10 + x + dx];
                    const float *w = sW1 + (dy * 3 + dx) * 32 + cg * 8;
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = fmaf(in, w[j], acc[j]);
                }
            float *dst = sA1 + (x >> 2) * A1P + (x & 3);
#pragma unroll
            for (int j = 0; j < 8; ++j) dst[((cg * 8 + j) * (VN_TB * 18) + yb) * 4] = fmaxf(acc[j], 0.f);
        }
        __syncthreads();
        // ---- conv2 (32->32, 18x8 -> 16x6) + ReLU: thread = (cout group of 8, board, output row), 6 px x 8 cout
        {
            const int cg = t >> 6, by = t & 63, b = by >> 4, y = by & 15;
            float acc[6][8];
#pragma unroll
            for (int p = 0; p < 6; ++p)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[p][j] = sB[32 + cg * 8 + j];
            for (int ci = 0; ci < 32; ++ci) {
#pragma unroll
                for (int dy = 0; dy < 3; ++dy) {
                    int rowi = (ci * (VN_TB * 18) + b * 18 + y + dy) * 4;
                    float4 l = *reinterpret_cast<const float4 *>(sA1 + rowi);
                    float4 r = *reinterpret_cast<const float4 *>(sA1 + A1P + rowi);
                    float in[8] = {l.x, l.y, l.z, l.w, r.x, r.y, r.z, r.w};
#pragma unroll
                    for (int dx = 0; dx < 3; ++dx) {
                        const float4 *wp = reinterpret_cast<const float4 *>(sW2 + (ci * 9 + dy * 3 + dx) * 32 + cg * 8);
                        float4 wa = wp[0], wb = wp[1];
                        float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
                        for (int p = 0; p < 6; ++p)
#pragma unroll
                            for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(in[p + dx], w[j], acc[p][j]);
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                int rowi = ((cg * 8 + j) * (VN_TB * 16) + b * 16 + y) * 4;
                *reinterpret_cast<float4 *>(sA2 + rowi) =
                    make_float4(fmaxf(acc[0][j], 0.f), fmaxf(acc[1][j], 0.f), fmaxf(acc[2][j], 0.f), fmaxf(acc[3][j], 0.f));
                *reinterpret_cast<float4 *>(sA2 + A2P + rowi) = make_float4(fmaxf(acc[4][j], 0.f), fmaxf(acc[5][j], 0.f), 0.f, 0.f);
            }
        }
        __syncthreads();
        if constexpr (DBG) {   // sA1 and sA2 stay unchanged until the next tile's first __syncthreads
            for (int i = t; i < VN_TB * VN_DBG_FLOATS; i += VN_THREADS) {
                const int b = i / VN_DBG_FLOATS, e = i - b * VN_DBG_FLOATS, ridx = tile * VN_TB + b;
                if (ridx >= n_req) continue;
                float v;
                if (e < VN_DBG_A1) {
                    const int c = e / 144, y = (e >> 3) % 18, x = e & 7;
                    v = sA1[(x >> 2) * A1P + ((c * (VN_TB * 18) + b * 18 + y) * 4 + (x & 3))];
                } else {
                    const int e2 = e - VN_DBG_A1, c = e2 / 96, y = (e2 / 6) % 16, x = e2 % 6;
                    v = sA2[(x >> 2) * A2P + ((c * (VN_TB * 16) + b * 16 + y) * 4 + (x & 3))];
                }
                dbg[(size_t)ridx * VN_DBG_FLOATS + e] = v;
            }
        }
        // ---- conv3 (32->32, 16x6 -> 14x4) + ReLU: thread = (cout group, board, output row < 14), 4 px x 8 cout
        {
            const int cg = t >> 6, by = t & 63, b = by >> 4, y = by & 15;
            const int ridx = tile * VN_TB + b;
            if (y < 14 && ridx < n_req) {
                float acc[4][8];
#pragma unroll
                for (int p = 0; p < 4; ++p)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[p][j] = sB[64 + cg * 8 + j];
                for (int ci = 0; ci < 32; ++ci) {
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy) {
                        int rowi = (ci * (VN_TB * 16) + b * 16 + y + dy) * 4;
                        float4 l = *reinterpret_cast<const float4 *>(sA2 + rowi);
                        float2 r = *reinterpret_cast<const float2 *>(sA2 + A2P + rowi);
                        float in[6] = {l.x, l.y, l.z, l.w, r.x, r.y};
#pragma unroll
                        for (int dx = 0; dx < 3; ++dx) {
                            const float4 *wp = reinterpret_cast<const float4 *>(sW3 + (ci * 9 + dy * 3 + dx) * 32 + cg * 8);
                            float4 wa = wp[0], wb = wp[1];
                            float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
                            for (int p = 0; p < 4; ++p)
#pragma unroll
                                for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(in[p + dx], w[j], acc[p][j]);
                        }
                    }
                }
                float4 *dst = reinterpret_cast<float4 *>(act3 + (size_t)ridx * 1792 + (y * 32 + cg * 8) * 4);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    dst[j] = make_float4(fmaxf(acc[0][j], 0.f), fmaxf(acc[1][j], 0.f), fmaxf(acc[2][j], 0.f), fmaxf(acc[3][j], 0.f));
            }
        }
    }
}

__global__ void __launch_bounds__(VN_THREADS, 1)
k_vn_conv(NetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M, float *act3) {
    vn_conv_body<false>(W, req, n_req_ptr, keys, M, act3, nullptr);
}
__global__ void __launch_bounds__(VN_THREADS, 1)
k_vn_conv_dbg(NetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M, float *act3, float *dbg) {
    vn_conv_body<true>(W, req, n_req_ptr, keys, M, act3, dbg);
}

// ---------------------------------------------------------------------------------------------------- fc1 + head
constexpr int FC_BM = 64, FC_BN = 256, FC_BK = 16, FC_THREADS = 256;

// With DBG, each row's fc1 accumulator (before the bias and the ReLU) is also written to dbg + ridx * 256 in torch column order
// (b200_debug_net_acts returns it).  Only k_vn_fc_dbg instantiates it.
template <bool DBG>
__device__ __forceinline__ void vn_fc_body(NetWeights W, const float *act3, const uint2 *req, const int32_t *n_req_ptr, float2 *eval_out,
                                           float *dbg) {
    __shared__ __align__(16) float sA[2][FC_BK][FC_BM];     // transposed: [k][row]
    __shared__ __align__(16) float sBm[2][FC_BK][FC_BN];
    const int n_req = *n_req_ptr;
    const int t = threadIdx.x, tx = t & 31, ty = t >> 5;
    const int n_tiles = (n_req + FC_BM - 1) / FC_BM;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int row0 = tile * FC_BM;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        // loaders: A: thread -> (row = t/4, k quad = t%4); B: 4 float4 per thread
        const int ar = t >> 2, ak = (t & 3) * 4;
        const bool arow_ok = row0 + ar < n_req;
        const float *aptr = act3 + (size_t)(row0 + ar) * 1792 + ak;
        float4 ra = arow_ok ? *reinterpret_cast<const float4 *>(aptr) : make_float4(0, 0, 0, 0);
        float4 rb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) rb[q] = *reinterpret_cast<const float4 *>(W.wfc1 + (size_t)(q * 4 + (t >> 6)) * 256 + (t & 63) * 4);
        int buf = 0;
        __syncthreads();
        for (int k0 = 0; k0 < 1792; k0 += FC_BK) {
            sA[buf][ak][ar] = ra.x; sA[buf][ak + 1][ar] = ra.y; sA[buf][ak + 2][ar] = ra.z; sA[buf][ak + 3][ar] = ra.w;
#pragma unroll
            for (int q = 0; q < 4; ++q) *reinterpret_cast<float4 *>(&sBm[buf][q * 4 + (t >> 6)][(t & 63) * 4]) = rb[q];
            __syncthreads();
            if (k0 + FC_BK < 1792) {
                ra = arow_ok ? *reinterpret_cast<const float4 *>(aptr + k0 + FC_BK) : make_float4(0, 0, 0, 0);
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    rb[q] = *reinterpret_cast<const float4 *>(W.wfc1 + (size_t)(k0 + FC_BK + q * 4 + (t >> 6)) * 256 + (t & 63) * 4);
            }
#pragma unroll
            for (int k = 0; k < FC_BK; ++k) {
                float4 a0 = *reinterpret_cast<const float4 *>(&sA[buf][k][ty * 8]);
                float4 a1 = *reinterpret_cast<const float4 *>(&sA[buf][k][ty * 8 + 4]);
                float4 b0 = *reinterpret_cast<const float4 *>(&sBm[buf][k][tx * 4]);
                float4 b1 = *reinterpret_cast<const float4 *>(&sBm[buf][k][128 + tx * 4]);
                float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            buf ^= 1;
        }
        // epilogue: bias + ReLU (model_vv.py:39-40), fc_out (:41), sigmoid (:42), affine (:51)
        float bias[8], wo0[8], wo1[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int col = (j < 4) ? tx * 4 + j : 128 + tx * 4 + (j - 4);
            bias[j] = W.bfc1[col]; wo0[j] = W.wout[col]; wo1[j] = W.wout[256 + col];
        }
        if constexpr (DBG) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = row0 + ty * 8 + i;
                if (r < n_req)
#pragma unroll
                    for (int j = 0; j < 8; ++j) dbg[(size_t)r * 256 + ((j < 4) ? tx * 4 + j : 128 + tx * 4 + (j - 4))] = acc[i][j];
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float p0 = 0.f, p1 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float h = fmaxf(acc[i][j] + bias[j], 0.f);
                p0 = fmaf(h, wo0[j], p0); p1 = fmaf(h, wo1[j], p1);
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                p0 += __shfl_xor_sync(0xffffffffu, p0, off);
                p1 += __shfl_xor_sync(0xffffffffu, p1, off);
            }
            int r = row0 + ty * 8 + i;
            if (tx == 0 && r < n_req) {
                float x0 = p0 + W.bout[0], x1 = p1 + W.bout[1];
                float s0 = 1.f / (1.f + expf(-x0)), s1 = 1.f / (1.f + expf(-x1));
                uint2 rq = req[r];
                eval_out[(size_t)rq.x * 8 + (rq.y >> 28)] =
                    make_float2(__fadd_rn(__fmul_rn(s0, W.ub[0]), W.lb[0]), __fadd_rn(__fmul_rn(s1, W.ub[1]), W.lb[1]));   // model_vv.py:51
            }
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(FC_THREADS)
k_vn_fc(NetWeights W, const float *act3, const uint2 *req, const int32_t *n_req_ptr, float2 *eval_out) {
    vn_fc_body<false>(W, act3, req, n_req_ptr, eval_out, nullptr);
}
__global__ void __launch_bounds__(FC_THREADS)
k_vn_fc_dbg(NetWeights W, const float *act3, const uint2 *req, const int32_t *n_req_ptr, float2 *eval_out, float *dbg) {
    vn_fc_body<true>(W, act3, req, n_req_ptr, eval_out, dbg);
}

}  // namespace b200
