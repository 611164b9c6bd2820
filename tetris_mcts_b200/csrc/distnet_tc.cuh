// distnet_tc.cuh — the reference's distributional value network (model/model_distributional.py:18-52) on Hopper tensor cores, built from
// the pieces of valuenet_tc.cuh (same fp16 x 2 operand split, same scaling, same no-swizzle K-major operand layouts, wgmma):
//
//   k_tdc_conv  persistent CTAs of TDC_WGS warpgroups, each carrying its own boards.  The 20x10 observation gets the reference's two empty
//               rows on top (22x10, model_distributional.py:27).  conv1 4x4 (1->32): im2col [19x8 grid = 152 rows][16 taps] built by the
//               warpgroup from the observation key, ONE K=16 wgmma per 64-row tile (three tiles).  conv2 4x4 (32->32) as a shift-GEMM on the
//               8-wide grid: A = act1 started dy*8 rows later, the four horizontal taps stacked along N = 128, 4 dy x 2 channel halves x 3 split
//               products = 24 wgmma (M=64, N=128, K=16) per tile; the epilogue sums the taps with three lane shuffles, applies bias +
//               LeakyReLU(0.01), re-splits and writes act2 (16x4 pixels x 32 channels = 2048 per board) to HBM in k_tdc_fc's tile layout.
//   k_tdc_fc    [R,2048] x [2048,128] like k_tc_fc (1-D TMA ring, producer warp + two consumer warpgroups); epilogue: bias + LeakyReLU ->
//               shared memory -> fc_v (128 x atoms, CUDA cores, one thread per board) -> softmax (model_distributional.py:47-50) -> dist[game][atoms].
#pragma once
#include "valuenet_tc.cuh"
#include "distnet_simt.cuh"

namespace b200 {

constexpr int TDC_WGS = 4;                       // warpgroups per CTA
constexpr int TDC_THREADS = TDC_WGS * 128;
constexpr int TDC_R = 152;                       // act1 rows per board: the 19x8 grid (conv2 reads rows m + dy*8 <= 127 + 24)
constexpr int TDC_WBLOCK = 2 * 2 * 128 * 16;     // one (dy, channel half) block of conv2: [weight split 2][chunk 2][n = dx*32 + cout][16 B]
constexpr int TDC_WBYTES = 8 * TDC_WBLOCK;       // 65536
constexpr int TDC_W1BYTES = 2 * 64 * 16;         // conv1: [chunk 2][n = split*32 + cout][16 B], k = tap = dy*4 + dx
constexpr int TDC_RUN = 4;
constexpr int TDC_ASLOT = 2 * 4 * TDC_R * 16;    // act1 of one board: [split][chunk 4][152 rows][16 B]
constexpr int TDC_IMROWS = 192;                  // three 64-row tiles (152 rows used)
constexpr int TDC_IMSLOT = 2 * TDC_IMROWS * 16;
constexpr int TDC_OFF_W2 = 0;
constexpr int TDC_OFF_W1 = TDC_OFF_W2 + TDC_WBYTES;
constexpr int TDC_OFF_A1 = TDC_OFF_W1 + TDC_W1BYTES;
constexpr int TDC_OFF_IM = TDC_OFF_A1 + TDC_WGS * TDC_ASLOT;
constexpr int TDC_OFF_BIAS = TDC_OFF_IM + TDC_WGS * TDC_IMSLOT;      // 64 floats, pre-scaled by TC_SCALE_A
constexpr int TDC_OFF_KEY = TDC_OFF_BIAS + 64 * 4;                   // TDC_WGS x 32 words: row table of the 22-row input (rows 0, 1 empty)
constexpr int TDC_SMEM = TDC_OFF_KEY + TDC_WGS * 32 * 4;
constexpr int DACT2_KCHUNKS = 256;               // 2048 / 8
static_assert(TDC_SMEM <= 227 * 1024, "k_tdc_conv shared memory");

struct DnTcWeights {
    const uint8_t *wc1;   // TDC_W1BYTES
    const uint8_t *wc2;   // TDC_WBYTES, already in the shared-memory layout
    const uint8_t *wfc;   // [split 2][k16 block 128][chunk 2][n 128][16 B]
};

// act2 in HBM, FC-tile layout: [split][tile of 128 boards][k chunk 256][board 128][8 fp16], k' = (y*4 + x)*32 + c
__device__ __forceinline__ size_t dact2_off(int split, int n_tiles, int ridx, int kchunk) {
    return ((((size_t)split * n_tiles + (ridx >> 7)) * DACT2_KCHUNKS + kchunk) * 128 + (ridx & 127)) * 16;
}

// conv2 on one 64-row tile = 24 wgmma of N = 128: for each (dy, channel half): a1*W1, a1*W2, a2*W1 into the same 128 columns
__device__ __forceinline__ void issue_dconv2(float (&d)[64], uint32_t a_addr, uint32_t w_addr) {
    const uint64_t a0 = gmma_desc(a_addr, TDC_R * 16, 128), b0 = gmma_desc(w_addr, 128 * 16, 128);
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const uint32_t a_hi = 2 * h * TDC_R + dy * 8, a_lo = a_hi + 4 * TDC_R;          // 16-byte units
            const uint32_t b_hi = (dy * 2 + h) * (TDC_WBLOCK / 16), b_lo = b_hi + 2 * 128;
            wgmma_n128(d, a0 + a_hi, b0 + b_hi, (dy | h) ? 1u : 0u);
            wgmma_n128(d, a0 + a_hi, b0 + b_lo, 1u);
            wgmma_n128(d, a0 + a_lo, b0 + b_hi, 1u);
        }
    }
}

__global__ void __launch_bounds__(TDC_THREADS, 1)
k_tdc_conv(DistNetWeights W, DnTcWeights TW, const uint2 *req, const int32_t *n_req_ptr, const uint32_t *keys, int M, uint8_t *act2, int n_tiles) {
    extern __shared__ __align__(128) uint8_t smem[];
    float *sB = reinterpret_cast<float *>(smem + TDC_OFF_BIAS);
    const int t = threadIdx.x, wg = t >> 7, wt = t & 127, w = wt >> 5, lane = t & 31;
    for (int i = t; i < TDC_WBYTES / 16; i += TDC_THREADS) reinterpret_cast<uint4 *>(smem + TDC_OFF_W2)[i] = reinterpret_cast<const uint4 *>(TW.wc2)[i];
    for (int i = t; i < TDC_W1BYTES / 16; i += TDC_THREADS) reinterpret_cast<uint4 *>(smem + TDC_OFF_W1)[i] = reinterpret_cast<const uint4 *>(TW.wc1)[i];
    for (int i = t; i < (TDC_OFF_BIAS - TDC_OFF_A1) / 16; i += TDC_THREADS) reinterpret_cast<uint4 *>(smem + TDC_OFF_A1)[i] = make_uint4(0, 0, 0, 0);
    // pre-scaled by 16: leaky(x * 2^-10 + b) * 16 == leaky(fma(x, 2^-6, 16 b)) bit for bit
    if (t < 32) { sB[t] = W.b1[t] * TC_SCALE_A; sB[32 + t] = W.b2[t] * TC_SCALE_A; }
    fence_async_smem();
    __syncthreads();
    const int n_req = *n_req_ptr;
    const int n_workers = (int)gridDim.x * TDC_WGS, wid = (int)blockIdx.x * TDC_WGS + wg;
    const int n_runs = (n_req + TDC_RUN - 1) / TDC_RUN;
    int n_local = 0;
    for (int run = wid; run < n_runs; run += n_workers) n_local += min(TDC_RUN, n_req - run * TDC_RUN);
    auto board_of = [&](int i) -> int { return ((i / TDC_RUN) * n_workers + wid) * TDC_RUN + (i % TDC_RUN); };
    uint8_t *act = smem + TDC_OFF_A1 + wg * TDC_ASLOT, *im = smem + TDC_OFF_IM + wg * TDC_IMSLOT;
    uint32_t *sKey = reinterpret_cast<uint32_t *>(smem + TDC_OFF_KEY) + wg * 32;
    const uint32_t s_act = smem_u32(act), s_im = smem_u32(im), s_w1 = smem_u32(smem + TDC_OFF_W1), s_w2 = smem_u32(smem + TDC_OFF_W2);
    const int qd = lane & 3, rl = lane >> 2;
    constexpr float K2 = TC_UNSCALE * TC_SCALE_A, K1 = TC_SCALE_A / TC_SCALE_W;
    constexpr int SPLIT = 4 * TDC_R * 16;
    auto fetch = [&](int i) -> uint32_t {                // lanes 0..11 of warp 0: the next board's key, in flight while this one is evaluated
        if (i >= n_local || lane >= 12) return 0u;
        const uint2 rq = req[board_of(i)];
        return keys[((size_t)rq.x * M + (rq.y & 0x0fffffffu)) * KEY_WORDS + lane];
    };
    uint32_t kw = w == 0 ? fetch(0) : 0u;
    for (int i = 0; i < n_local; ++i) {
        const int ridx = board_of(i);
        if (w == 0) {
            // lane l < 22 holds input row l = board row l - 2 (rows 0, 1: the reference's padding): settled cells in bits 0..9, piece cells in 16..25
            const int br = lane - 2;
            const uint32_t rowpair = __shfl_sync(0xffffffffu, kw, (br >> 1) & 15), pcs = __shfl_sync(0xffffffffu, kw, 10);
            uint32_t tab = (rowpair >> ((br & 1) * 16)) & 0x3ffu;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t cell = (pcs >> (8 * k)) & 0xffu, pr = (cell * 205u) >> 11, pcol = cell - pr * 10u;
                tab |= ((int)pr == br ? 1u : 0u) << (16 + pcol);
            }
            if (br < 0 || br >= 20) tab = 0u;
            kw = fetch(i + 1);
            if (lane < 22) sKey[lane] = tab;
        }
        wg_sync(wg);
        // im2col of conv1 (fp16, exact {-1,0,1}): row p = y*8 + x of the 19x8 output grid, k = tap = dy*4 + dx; taps 0..7 in the first k chunk
        for (int p = wt; p < TDC_R; p += 128) {
            const int y = p >> 3, x = p & 7;
            uint32_t hv[16];
#pragma unroll
            for (int dy = 0; dy < 4; ++dy) {
                const uint32_t rw = sKey[y + dy] >> x;
#pragma unroll
                for (int dx = 0; dx < 4; ++dx)       // 1 settled, -1 falling piece, 0 empty; columns >= 10 (x = 7) read zero bits
                    hv[dy * 4 + dx] = ((rw >> dx) & 1u) * 0x3C00u | ((rw >> (16 + dx)) & 1u & (x + dx < 10 ? 1u : 0u)) * 0xBC00u;
            }
            *reinterpret_cast<uint4 *>(im + p * 16) =
                make_uint4(hv[0] | (hv[1] << 16), hv[2] | (hv[3] << 16), hv[4] | (hv[5] << 16), hv[6] | (hv[7] << 16));
            *reinterpret_cast<uint4 *>(im + TDC_IMROWS * 16 + p * 16) =
                make_uint4(hv[8] | (hv[9] << 16), hv[10] | (hv[11] << 16), hv[12] | (hv[13] << 16), hv[14] | (hv[15] << 16));
        }
        fence_async_smem();
        wg_sync(wg);
        // ---- conv1 (model_distributional.py:20): im2col [192 x 16] x W1 [16 x 64], three 64-row tiles; epilogue: bias + LeakyReLU + split -> act1
#pragma unroll 1
        for (int mt = 0; mt < 3; ++mt) {
            float d[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) d[k] = 0.f;
            wgmma_fence();
            wgmma_n64(d, gmma_desc(s_im + mt * 1024, TDC_IMROWS * 16, 128), gmma_desc(s_w1, 64 * 16, 128), 0u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(d);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = mt * 64 + 16 * w + 8 * h + rl;
                if (r < TDC_R) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int c = 8 * j + 2 * qd;
                        const float o0 = leaky(fmaf(d[4 * (j + 4) + 2 * h] + d[4 * j + 2 * h], K1, sB[c]));
                        const float o1 = leaky(fmaf(d[4 * (j + 4) + 2 * h + 1] + d[4 * j + 2 * h + 1], K1, sB[c + 1]));
                        uint32_t hi, lo;
                        split2(o0, o1, hi, lo);
                        uint8_t *dst = act + (j * TDC_R + r) * 16 + qd * 4;
                        *reinterpret_cast<uint32_t *>(dst) = hi;
                        *reinterpret_cast<uint32_t *>(dst + SPLIT) = lo;
                    }
                }
            }
        }
        fence_async_smem();
        wg_sync(wg);
        // ---- conv2 (model_distributional.py:22): act1 on the 19x8 grid; epilogue: dx sum + bias + LeakyReLU + split -> act2 in HBM
#pragma unroll 1
        for (int mt = 0; mt < 2; ++mt) {
            float d[64];
#pragma unroll
            for (int k = 0; k < 64; ++k) d[k] = 0.f;
            wgmma_fence();
            issue_dconv2(d, s_act + mt * 1024, s_w2);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(d);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int y = mt * 8 + 2 * w + h, x = rl;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {                // out[p] = D'[p][0] + D'[p+1][1] + D'[p+2][2] + D'[p+3][3]
                        const int k = 4 * j + 2 * h + e;
                        const float s1 = __shfl_down_sync(0xffffffffu, d[16 + k], 4), s2 = __shfl_down_sync(0xffffffffu, d[32 + k], 8),
                                    s3 = __shfl_down_sync(0xffffffffu, d[48 + k], 12);
                        o[e] = leaky(fmaf(((s3 + s2) + s1) + d[k], K2, sB[32 + 8 * j + 2 * qd + e]));
                    }
                    uint32_t hi, lo;
                    split2(o[0], o[1], hi, lo);
                    if (x < 4) {
                        const int kc = (y * 4 + x) * 4 + j;
                        *reinterpret_cast<uint32_t *>(act2 + dact2_off(0, n_tiles, ridx, kc) + qd * 4) = hi;
                        *reinterpret_cast<uint32_t *>(act2 + dact2_off(1, n_tiles, ridx, kc) + qd * 4) = lo;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------- fc1 + fc_v + softmax
constexpr int TDF_CONSUMERS = 2;            // warpgroups 0-1: MMA + epilogue, 64 boards of the 128-board tile each
constexpr int TDF_PRODUCER = TDF_CONSUMERS * 4;
constexpr int TDF_THREADS = TDF_CONSUMERS * 128 + 32;
constexpr int TDF_STAGES = 6;
constexpr int TDF_A_BYTES = 2 * 128 * 16;   // one split of one k16 block of the A tile
constexpr int TDF_B_BYTES = 2 * 128 * 16;
constexpr int TDF_STAGE = 2 * TDF_A_BYTES + 2 * TDF_B_BYTES;   // 16384
constexpr int TDF_KBLOCKS = 128;            // 2048 / 16
constexpr int TDF_ATOMS = 64;               // fc_v columns carried per thread (atoms <= 64, the rest zero)
constexpr int TDF_HSTRIDE = 129;            // fc1 activations in shared memory: [board][128 + 1] (the pad keeps the row-per-thread reads conflict free)
constexpr int TDF_OFF_BAR = TDF_STAGES * TDF_STAGE;
constexpr int TDF_OFF_EPI = TDF_OFF_BAR + 256;                 // bias[128] | wv[128][64] | bv[64] | h[2][64][129]
static_assert(2 * TDF_STAGES * 8 <= 256, "barrier block overflows into the epilogue constants");
constexpr int TDF_SMEM = TDF_OFF_EPI + (128 + 128 * TDF_ATOMS + TDF_ATOMS + TDF_CONSUMERS * 64 * TDF_HSTRIDE) * 4;
static_assert(TDF_SMEM <= 227 * 1024, "k_tdc_fc shared memory");

__global__ void __launch_bounds__(TDF_THREADS, 1)
k_tdc_fc(DistNetWeights W, DnTcWeights TW, const uint8_t *act2, int n_tiles_alloc, const uint2 *req, const int32_t *n_req_ptr, float *out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + TDF_OFF_BAR);
    uint64_t *empty = full + TDF_STAGES;
    float *sBias = reinterpret_cast<float *>(smem + TDF_OFF_EPI), *sWv = sBias + 128, *sBv = sWv + 128 * TDF_ATOMS, *sH = sBv + TDF_ATOMS;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31, atoms = W.atoms;
    for (int i = t; i < 128; i += TDF_THREADS) sBias[i] = W.bf1[i];
    for (int i = t; i < 128 * TDF_ATOMS; i += TDF_THREADS) { const int k = i / TDF_ATOMS, a = i - k * TDF_ATOMS; sWv[i] = a < atoms ? W.wfv[(size_t)k * atoms + a] : 0.f; }
    if (t < TDF_ATOMS) sBv[t] = t < atoms ? W.bfv[t] : 0.f;
    if (t == 0) {
        for (int i = 0; i < TDF_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TDF_CONSUMERS); }
        fence_barrier_init();
    }
    __syncthreads();
    const int n_req = *n_req_ptr;
    const int n_tiles = (n_req + 127) >> 7;
    if (warp == TDF_PRODUCER) {
        if (lane == 0) {   // ===== producer: bulk copies of the pre-laid-out operand blocks
            int stage = 0; uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                for (int j = 0; j < TDF_KBLOCKS; ++j) {
                    mbar_wait(&empty[stage], ph ^ 1);
                    mbar_expect_tx(&full[stage], TDF_STAGE);
                    uint8_t *dst = smem + stage * TDF_STAGE;
#pragma unroll
                    for (int s = 0; s < 2; ++s) {
                        bulk_g2s(dst + s * TDF_A_BYTES, act2 + (((size_t)s * n_tiles_alloc + tile) * DACT2_KCHUNKS + 2 * j) * 2048, TDF_A_BYTES, &full[stage]);
                        bulk_g2s(dst + 2 * TDF_A_BYTES + s * TDF_B_BYTES, TW.wfc + ((size_t)s * TDF_KBLOCKS + j) * TDF_B_BYTES, TDF_B_BYTES, &full[stage]);
                    }
                    if (++stage == TDF_STAGES) { stage = 0; ph ^= 1; }
                }
            }
        }
    } else {   // ===== consumers: D[64 x 128] += A[64 x 16] * B[128 x 16]^T per warpgroup, three split terms per k block
        const int wg = t >> 7, wt = t & 127, w = warp & 3, qd = lane & 3, rl = lane >> 2;
        float *hrow = sH + wg * 64 * TDF_HSTRIDE;
        int stage = 0; uint32_t ph = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            float d[64];
#pragma unroll
            for (int k = 0; k < 64; ++k) d[k] = 0.f;
            int prev = -1;
            for (int j = 0; j < TDF_KBLOCKS; ++j) {
                mbar_wait(&full[stage], ph);
                const uint32_t sbase = smem_u32(smem + stage * TDF_STAGE);
                wgmma_fence();
#pragma unroll
                for (int term = 0; term < 3; ++term) {   // a1*b2, a2*b1, a1*b1 (small terms first)
                    const int sa = term == 1 ? 1 : 0, sb = term == 0 ? 1 : 0;
                    const uint64_t ad = gmma_desc(sbase + sa * TDF_A_BYTES + wg * 1024, 128 * 16, 128);
                    const uint64_t bd = gmma_desc(sbase + 2 * TDF_A_BYTES + sb * TDF_B_BYTES, 128 * 16, 128);
                    wgmma_n128(d, ad, bd, (j | term) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();
                if (prev >= 0 && wt == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == TDF_STAGES) { stage = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(d);
            if (wt == 0) mbar_arrive(&empty[prev]);
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * j + 2 * qd + e;
                        hrow[(16 * w + 8 * h + rl) * TDF_HSTRIDE + c] = leaky(d[4 * j + 2 * h + e] * TC_UNSCALE + sBias[c]);   // model_distributional.py:43-44
                    }
            wg_sync(wg);
            const int ridx = tile * 128 + wg * 64 + wt;
            if (wt < 64 && ridx < n_req) {
                float lg[TDF_ATOMS];
#pragma unroll
                for (int a = 0; a < TDF_ATOMS; ++a) lg[a] = sBv[a];
#pragma unroll 1
                for (int c = 0; c < 128; ++c) {
                    const float hv = hrow[wt * TDF_HSTRIDE + c];
                    const float4 *wv = reinterpret_cast<const float4 *>(sWv + c * TDF_ATOMS);
#pragma unroll
                    for (int a4 = 0; a4 < TDF_ATOMS / 4; ++a4) {                        // :45 (ascending k, like the CUDA-core kernel)
                        const float4 w4 = wv[a4];
                        lg[4 * a4] = fmaf(hv, w4.x, lg[4 * a4]); lg[4 * a4 + 1] = fmaf(hv, w4.y, lg[4 * a4 + 1]);
                        lg[4 * a4 + 2] = fmaf(hv, w4.z, lg[4 * a4 + 2]); lg[4 * a4 + 3] = fmaf(hv, w4.w, lg[4 * a4 + 3]);
                    }
                }
                float mx = -INFINITY;                                                  // F.softmax(x, 1), :47-50
#pragma unroll
                for (int a = 0; a < TDF_ATOMS; ++a) if (a < atoms) mx = fmaxf(mx, lg[a]);
                float sum = 0.f;
#pragma unroll
                for (int a = 0; a < TDF_ATOMS; ++a) if (a < atoms) { lg[a] = expf(lg[a] - mx); sum += lg[a]; }
                float *dst = out + (size_t)req[ridx].x * atoms;
#pragma unroll
                for (int a = 0; a < TDF_ATOMS; ++a) if (a < atoms) dst[a] = lg[a] / sum;
            }
            wg_sync(wg);                                 // h is rewritten by the next tile's epilogue
        }
    }
}

// ---------------------------------------------------------------------------------------------------- host side
struct DnTcState {
    uint8_t *d_w = nullptr;      // wc1 | wc2 | wfc
    DnTcWeights TW{};
    uint8_t *d_act2 = nullptr; size_t tiles = 0;
};

// w = the state_dict-order weight vector of model_distributional.py (see dn_relayout).  Pure re-layout + fp16 splitting.
static int dn_tc_prepare(void **state, const float *w, int atoms, cudaStream_t stream) {
    DnTcState *st = (DnTcState *)*state;
    if (!st) { st = new DnTcState(); *state = st; }
    const float *c1w = w, *c2w = c1w + 512 + 32, *f1w = c2w + 16384 + 32;
    (void)atoms;
    const size_t fc_bytes = (size_t)2 * TDF_KBLOCKS * TDF_B_BYTES;
    std::vector<uint8_t> h(TDC_W1BYTES + (size_t)TDC_WBYTES + fc_bytes);
    uint16_t *p1 = reinterpret_cast<uint16_t *>(h.data()), *p2 = reinterpret_cast<uint16_t *>(h.data() + TDC_W1BYTES);
    uint16_t *pf = reinterpret_cast<uint16_t *>(h.data() + TDC_W1BYTES + TDC_WBYTES);
    for (int c2 = 0; c2 < 2; ++c2)                               // conv1: [chunk][n = split*32 + cout][8], k = tap = dy*4 + dx
        for (int n = 0; n < 32; ++n)
            for (int e = 0; e < 8; ++e) {
                uint16_t s2[2];
                host_split2(c1w[n * 16 + 8 * c2 + e] * TC_SCALE_W, s2);
                for (int s = 0; s < 2; ++s) p1[((size_t)c2 * 64 + s * 32 + n) * 8 + e] = s2[s];
            }
    for (int dy = 0; dy < 4; ++dy)                               // conv2: [(dy, half)][split][chunk][n = dx*32 + cout][8]
        for (int hh = 0; hh < 2; ++hh)
            for (int c2 = 0; c2 < 2; ++c2)
                for (int dx = 0; dx < 4; ++dx)
                    for (int n = 0; n < 32; ++n)
                        for (int e = 0; e < 8; ++e) {
                            const int ci = 16 * hh + 8 * c2 + e;
                            uint16_t s2[2];
                            host_split2(c2w[(n * 32 + ci) * 16 + dy * 4 + dx] * TC_SCALE_W, s2);
                            for (int s = 0; s < 2; ++s) p2[(((((size_t)(dy * 2 + hh)) * 2 + s) * 2 + c2) * 128 + dx * 32 + n) * 8 + e] = s2[s];
                        }
    for (int j = 0; j < TDF_KBLOCKS; ++j)                        // fc1: k' = pixel*32 + channel, pixel = y*4 + x; torch k = c*64 + pixel
        for (int c2 = 0; c2 < 2; ++c2)
            for (int n = 0; n < 128; ++n)
                for (int e = 0; e < 8; ++e) {
                    const int kp = j * 16 + c2 * 8 + e, p = kp >> 5, c = kp & 31;
                    uint16_t s2[2];
                    host_split2(f1w[(size_t)n * 2048 + c * 64 + p] * TC_SCALE_W, s2);
                    for (int s = 0; s < 2; ++s) pf[((((size_t)s * TDF_KBLOCKS + j) * 2 + c2) * 128 + n) * 8 + e] = s2[s];
                }
    if (!st->d_w && cudaMalloc(&st->d_w, h.size()) != cudaSuccess) return 1;
    if (cudaMemcpyAsync(st->d_w, h.data(), h.size(), cudaMemcpyHostToDevice, stream) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return 1;
    st->TW.wc1 = st->d_w; st->TW.wc2 = st->d_w + TDC_W1BYTES; st->TW.wfc = st->TW.wc2 + TDC_WBYTES;
    if (cudaFuncSetAttribute(k_tdc_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, TDC_SMEM) != cudaSuccess) return 1;
    if (cudaFuncSetAttribute(k_tdc_fc, cudaFuncAttributeMaxDynamicSharedMemorySize, TDF_SMEM) != cudaSuccess) return 1;
    return 0;
}

static int dn_tc_ensure_act2(DnTcState *st, size_t max_rows, cudaStream_t stream, bool *moved) {
    size_t tiles = (max_rows + 127) / 128;
    if (st->tiles >= tiles) return 0;
    if (st->d_act2) { cudaStreamSynchronize(stream); cudaFree(st->d_act2); st->d_act2 = nullptr; if (moved) *moved = true; }
    size_t bytes = (size_t)2 * tiles * DACT2_KCHUNKS * 2048;
    if (cudaMalloc(&st->d_act2, bytes) != cudaSuccess) return 1;
    cudaMemsetAsync(st->d_act2, 0, bytes, stream);
    st->tiles = tiles;
    return 0;
}

static void dn_tc_destroy(void *state) {
    DnTcState *st = (DnTcState *)state;
    if (!st) return;
    cudaFree(st->d_w); cudaFree(st->d_act2);
    delete st;
}

}  // namespace b200
