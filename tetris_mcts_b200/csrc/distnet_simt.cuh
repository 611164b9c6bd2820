// distnet_simt.cuh — forward pass of the reference's distributional value network (model/model_distributional.py:18-52):
// conv 4x4 (1->32) -> LeakyReLU(0.01) -> conv 4x4 (32->32) -> LeakyReLU -> flatten -> fc 128 -> LeakyReLU -> fc atoms -> softmax.
// The reference hard-codes a 22x10 input (model_distributional.py:27), so the 20x10 observation gets two empty rows on top;
// conv1 -> 19x7, conv2 -> 16x4, flatten 2048 in NCHW order.  fp32 CUDA cores: this network only serves BASELINE config 5
// (one board per simulation per game), a small fraction of the ValueSimLP traffic.
#pragma once
#include "search_dev.cuh"

namespace b200 {

struct DistNetWeights {
    const float *w1;    // [16][32]   tap-major, cout contiguous
    const float *w2;    // [512][32]  k = ci*16 + dy*4 + dx, cout contiguous
    const float *b1, *b2;
    const float *wf1;   // [2048][128] k-major (torch k = c*64 + y*4 + x), n contiguous
    const float *bf1;   // [128]
    const float *wfv;   // [128][atoms] k-major
    const float *bfv;   // [atoms]
    int atoms;
};

constexpr int DN_THREADS = 256;
constexpr int DN_CONV_SMEM = (512 * 32 + 16 * 32 + 64 + 220 + 32 * 136) * 4;
constexpr int DN_FC_ROWS = 8;
constexpr int DN_FC_SMEM = (DN_FC_ROWS * 2048 + DN_FC_ROWS * 128 + DN_FC_ROWS * 64) * 4;

static void dn_relayout(const float *w, int atoms, std::vector<float> &h) {
    const float *c1w = w, *c1b = c1w + 512, *c2w = c1b + 32, *c2b = c2w + 16384, *f1w = c2b + 32, *f1b = f1w + 128 * 2048;
    const float *fvw = f1b + 128, *fvb = fvw + (size_t)atoms * 128;
    h.assign(512 + 16384 + 64 + (size_t)2048 * 128 + 128 + (size_t)128 * atoms + atoms, 0.f);
    float *p = h.data();
    float *w1 = p; p += 512; float *w2 = p; p += 16384; float *b12 = p; p += 64; float *wf1 = p; p += (size_t)2048 * 128;
    float *bf1 = p; p += 128; float *wfv = p; p += (size_t)128 * atoms; float *bfv = p;
    for (int co = 0; co < 32; ++co)
        for (int tap = 0; tap < 16; ++tap) w1[tap * 32 + co] = c1w[co * 16 + tap];
    for (int co = 0; co < 32; ++co)
        for (int ci = 0; ci < 32; ++ci)
            for (int tap = 0; tap < 16; ++tap) w2[(ci * 16 + tap) * 32 + co] = c2w[(co * 32 + ci) * 16 + tap];
    for (int i = 0; i < 32; ++i) { b12[i] = c1b[i]; b12[32 + i] = c2b[i]; }
    for (int n = 0; n < 128; ++n)
        for (int k = 0; k < 2048; ++k) wf1[(size_t)k * 128 + n] = f1w[(size_t)n * 2048 + k];
    for (int n = 0; n < 128; ++n) bf1[n] = f1b[n];
    for (int a = 0; a < atoms; ++a)
        for (int k = 0; k < 128; ++k) wfv[(size_t)k * atoms + a] = fvw[(size_t)a * 128 + k];
    for (int a = 0; a < atoms; ++a) bfv[a] = fvb[a];
}

static DistNetWeights dn_pointers(const float *d, int atoms) {
    DistNetWeights W;
    W.w1 = d; W.w2 = d + 512; W.b1 = d + 512 + 16384; W.b2 = W.b1 + 32; W.wf1 = W.b1 + 64; W.bf1 = W.wf1 + (size_t)2048 * 128;
    W.wfv = W.bf1 + 128; W.bfv = W.wfv + (size_t)128 * atoms; W.atoms = atoms;
    return W;
}

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : 0.01f * x; }

__global__ void k_dn_req_rows(uint2 *req, int k) {   // standalone inference: request i writes output row i
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k) req[i] = make_uint2((uint32_t)i, (uint32_t)i);
}

// conv stack: persistent CTAs, one board per pass; act2 [request][2048] in NCHW flatten order.  With DBG, each board's act1 [32][19][7] is
// also copied to dbg + ridx * DN_DBG_A1 once conv1 has finished (b200_debug_net_acts returns it).  Only k_dn_conv_dbg instantiates it.
constexpr int DN_DBG_A1 = 32 * 133;

template <bool DBG>
__device__ __forceinline__ void dn_conv_body(DistNetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M, float *act,
                                             float *dbg) {
    extern __shared__ __align__(16) float sm[];
    float *sW2 = sm, *sW1 = sW2 + 512 * 32, *sB = sW1 + 16 * 32, *sIn = sB + 64, *sA1 = sIn + 220;   // sA1 [32][136] (19x7 = 133 used)
    const int t = threadIdx.x;
    for (int i = t; i < 512 * 32; i += DN_THREADS) sW2[i] = W.w2[i];
    for (int i = t; i < 512; i += DN_THREADS) sW1[i] = W.w1[i];
    if (t < 64) sB[t] = W.b1[t];
    const int n_req = *n_req_ptr;
    for (int ridx = blockIdx.x; ridx < n_req; ridx += gridDim.x) {
        __syncthreads();
        uint2 rq = req[ridx];
        const uint32_t *k = keys + ((size_t)rq.x * M + (rq.y & 0x0fffffffu)) * KEY_WORDS;
        if (t < 220) {
            float v = 0.f;
            if (t >= 20) {
                const int cell = t - 20, r = cell / 10, c = cell - r * 10;
                v = (float)((k[r >> 1] >> ((r & 1) * 16 + c)) & 1u);
                uint32_t pc = k[10], ci = (uint32_t)cell;
                if ((pc & 0xffu) == ci || ((pc >> 8) & 0xffu) == ci || ((pc >> 16) & 0xffu) == ci || (pc >> 24) == ci) v = -1.f;
            }
            sIn[t] = v;
        }
        __syncthreads();
        for (int task = t; task < 133 * 4; task += DN_THREADS) {      // conv1: (pixel of 19x7, 8-cout chunk)
            const int cq = task / 133, pix = task - cq * 133, y = pix / 7, x = pix - y * 7;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = sB[cq * 8 + j];
#pragma unroll
            for (int dy = 0; dy < 4; ++dy)
#pragma unroll
                for (int dx = 0; dx < 4; ++dx) {
                    const float in = sIn[(y + dy) * 10 + x + dx];
                    const float *w = sW1 + (dy * 4 + dx) * 32 + cq * 8;
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[j] = fmaf(in, w[j], acc[j]);
                }
#pragma unroll
            for (int j = 0; j < 8; ++j) sA1[(cq * 8 + j) * 136 + pix] = leaky(acc[j]);
        }
        __syncthreads();
        if constexpr (DBG) {   // sA1 stays unchanged until the next board's first __syncthreads
            for (int i = t; i < DN_DBG_A1; i += DN_THREADS) dbg[(size_t)ridx * DN_DBG_A1 + i] = sA1[(i / 133) * 136 + i % 133];
        }
        {   // conv2: thread = (pixel of 16x4, 8-cout chunk): 64 x 4 = 256 threads
            const int cq = t >> 6, pix = t & 63, y = pix >> 2, x = pix & 3;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] = sB[32 + cq * 8 + j];
            for (int ci = 0; ci < 32; ++ci) {
#pragma unroll
                for (int dy = 0; dy < 4; ++dy)
#pragma unroll
                    for (int dx = 0; dx < 4; ++dx) {
                        const float in = sA1[ci * 136 + (y + dy) * 7 + x + dx];
                        const float4 *w = reinterpret_cast<const float4 *>(sW2 + (ci * 16 + dy * 4 + dx) * 32 + cq * 8);
                        const float4 wa = w[0], wb = w[1];
                        acc[0] = fmaf(in, wa.x, acc[0]); acc[1] = fmaf(in, wa.y, acc[1]); acc[2] = fmaf(in, wa.z, acc[2]); acc[3] = fmaf(in, wa.w, acc[3]);
                        acc[4] = fmaf(in, wb.x, acc[4]); acc[5] = fmaf(in, wb.y, acc[5]); acc[6] = fmaf(in, wb.z, acc[6]); acc[7] = fmaf(in, wb.w, acc[7]);
                    }
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) act[(size_t)ridx * 2048 + (cq * 8 + j) * 64 + pix] = leaky(acc[j]);
        }
    }
}

__global__ void __launch_bounds__(DN_THREADS) k_dn_conv(DistNetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M,
                                                       float *act) {
    dn_conv_body<false>(W, req, n_req_ptr, keys, M, act, nullptr);
}
__global__ void __launch_bounds__(DN_THREADS) k_dn_conv_dbg(DistNetWeights W, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys,
                                                           int M, float *act, float *dbg) {
    dn_conv_body<true>(W, req, n_req_ptr, keys, M, act, dbg);
}

// fc1 + LeakyReLU + fc_v + softmax; DN_FC_ROWS boards per CTA pass; output row = req.x (the game) * atoms.  With DBG, each row's fc1
// accumulator (bias included, before the LeakyReLU) is also written to dbg_fc + ridx * 128, and its logits (before the softmax overwrites
// them) to dbg_lg + ridx * atoms (b200_debug_net_acts returns both).  Only k_dn_fc_dbg instantiates it.
template <bool DBG>
__device__ __forceinline__ void dn_fc_body(DistNetWeights W, const float *act, const uint2 *req, const int32_t *n_req_ptr, float *out, float *dbg_fc,
                                           float *dbg_lg) {
    extern __shared__ __align__(16) float sm[];
    float *sA = sm, *sH = sA + DN_FC_ROWS * 2048, *sL = sH + DN_FC_ROWS * 128;
    const int t = threadIdx.x, n_req = *n_req_ptr, atoms = W.atoms;
    for (int base = blockIdx.x * DN_FC_ROWS; base < n_req; base += gridDim.x * DN_FC_ROWS) {
        const int rows = min(DN_FC_ROWS, n_req - base);
        __syncthreads();
        for (int i = t; i < rows * 2048; i += DN_THREADS) sA[i] = act[(size_t)base * 2048 + i];
        __syncthreads();
        {   // fc1: thread = (output n = t % 128, row half = t / 128): 4 rows each
            const int n = t & 127, r0 = (t >> 7) * 4;
            float acc[4] = {W.bf1[n], W.bf1[n], W.bf1[n], W.bf1[n]};
            for (int k = 0; k < 2048; ++k) {
                const float w = W.wf1[(size_t)k * 128 + n];
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r] = fmaf(sA[(r0 + r) * 2048 + k], w, acc[r]);
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) sH[(r0 + r) * 128 + n] = leaky(acc[r]);
            if constexpr (DBG) {
#pragma unroll
                for (int r = 0; r < 4; ++r)
                    if (r0 + r < rows) dbg_fc[(size_t)(base + r0 + r) * 128 + n] = acc[r];
            }
        }
        __syncthreads();
        for (int task = t; task < rows * atoms; task += DN_THREADS) {     // fc_v logits
            const int r = task / atoms, a = task - r * atoms;
            float acc = W.bfv[a];
            for (int k = 0; k < 128; ++k) acc = fmaf(sH[r * 128 + k], W.wfv[(size_t)k * atoms + a], acc);
            sL[r * 64 + a] = acc;
            if constexpr (DBG) dbg_lg[(size_t)(base + r) * atoms + a] = acc;
        }
        __syncthreads();
        if (t < rows) {                                                    // softmax (F.softmax(x, 1), model_distributional.py:47-50)
            float mx = -INFINITY;
            for (int a = 0; a < atoms; ++a) mx = fmaxf(mx, sL[t * 64 + a]);
            float sum = 0.f;
            for (int a = 0; a < atoms; ++a) { float e = expf(sL[t * 64 + a] - mx); sL[t * 64 + a] = e; sum += e; }
            float *dst = out + (size_t)req[base + t].x * atoms;
            for (int a = 0; a < atoms; ++a) dst[a] = sL[t * 64 + a] / sum;
        }
    }
}

__global__ void __launch_bounds__(DN_THREADS) k_dn_fc(DistNetWeights W, const float *act, const uint2 *req, const int32_t *n_req_ptr, float *out) {
    dn_fc_body<false>(W, act, req, n_req_ptr, out, nullptr, nullptr);
}
__global__ void __launch_bounds__(DN_THREADS) k_dn_fc_dbg(DistNetWeights W, const float *act, const uint2 *req, const int32_t *n_req_ptr, float *out,
                                                         float *dbg_fc, float *dbg_lg) {
    dn_fc_body<true>(W, act, req, n_req_ptr, out, dbg_fc, dbg_lg);
}

}  // namespace b200
