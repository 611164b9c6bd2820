// ext_eval.cuh — the caller-supplied evaluator (B200_EVAL_EXTERNAL): the kernels that hand one simulation step's evaluation requests to
// the caller as boards and put the caller's outputs where the backup reads them (A.eval_out / A.dist_eval).
#pragma once
#include "search_dev.cuh"

namespace b200 {

constexpr int EXT_ORDER_THREADS = 1024;

// One cell of the board Model_VV.inference sees for observation key k (model_vv.py:212): the board bit, or -1 where one of the four
// falling-piece cells lies.  The rule k_vn_conv applies to its input tile.
__device__ __forceinline__ int ext_cell(const uint32_t *k, int cell) {
    const uint32_t pc = k[10], c = (uint32_t)cell;
    if ((pc & 0xffu) == c || ((pc >> 8) & 0xffu) == c || ((pc >> 16) & 0xffu) == c || (pc >> 24) == c) return -1;
    const int r = cell / 10, x = cell % 10;
    return (int)((k[r >> 1] >> ((r & 1) * 16 + x)) & 1u);
}

// The step's requests (A.req, in atomicAdd order) -> rows[0 .. *n_rows) in ascending (game, slot) order, in the request format
// {game, obs | slot << 28}.  One CTA: mark[g*8 + slot] = obs + 1, then a scan over games in a fixed order; the marks are cleared as they
// are read, so mark[] is all zero between steps.  Each (game, slot) is requested at most once per step.
__global__ void __launch_bounds__(EXT_ORDER_THREADS) k_ext_order(Arena A, int32_t *mark, uint2 *rows, int32_t *n_rows) {
    __shared__ int s_warp[EXT_ORDER_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    const int n = *A.n_req;
    for (int i = t; i < n; i += EXT_ORDER_THREADS) {
        const uint2 r = A.req[i];
        mark[(size_t)r.x * 8 + (r.y >> 28)] = (int32_t)(r.y & 0x0fffffffu) + 1;
    }
    __syncthreads();
    const int per = (A.G + EXT_ORDER_THREADS - 1) / EXT_ORDER_THREADS;     // thread t scans games [g0, g1)
    const int g0 = min(t * per, A.G), g1 = min(g0 + per, A.G);
    int cnt = 0;
    for (int g = g0; g < g1; ++g)
        for (int s = 0; s < 8; ++s) cnt += mark[(size_t)g * 8 + s] != 0;
    int incl = cnt;                                                      // exclusive scan of cnt over the CTA
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += y; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int base = incl - cnt, total = 0;
    for (int w = 0; w < EXT_ORDER_THREADS / 32; ++w) { if (w < wid) base += s_warp[w]; total += s_warp[w]; }
    for (int g = g0; g < g1; ++g)
        for (int s = 0; s < 8; ++s) {
            int32_t &m = mark[(size_t)g * 8 + s];
            if (m) { rows[base++] = make_uint2((uint32_t)g, (uint32_t)(m - 1) | ((uint32_t)s << 28)); m = 0; }
        }
    if (t == 0) *n_rows = total;
}

// boards[row][200] (= NCHW [n,1,20,10]) of the ordered rows, as int8 or float32; ids[row] = game * 8 + slot (ids may be nullptr)
template <typename T>
__global__ void k_ext_boards(Arena A, const uint2 *rows, const int32_t *n_rows, T *boards, int32_t *ids) {
    const size_t n = (size_t)*n_rows * 200;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int row = (int)(i / 200), cell = (int)(i % 200);
        const uint2 r = rows[row];
        boards[i] = (T)ext_cell(A.key + node_at(A, (int)r.x, (int)(r.y & 0x0fffffffu)) * KEY_WORDS, cell);
        if (ids && cell == 0) ids[row] = (int32_t)(r.x * 8 + (r.y >> 28));
    }
}

// out[row][cols] (fp32, row-major) -> eval_out[g*8 + slot] = (v, var) (cols = 2), or dist_eval[g*cols + b] (distributional mode).
// Values are copied as they are, NaN included.
__global__ void k_ext_scatter(Arena A, const uint2 *rows, const int32_t *n_rows, const float *out, int cols) {
    const size_t n = (size_t)*n_rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int row = (int)(i / cols), c = (int)(i % cols);
        const uint2 r = rows[row];
        if (A.mode == MODE_DIST) A.dist_eval[(size_t)r.x * cols + c] = out[i];
        else reinterpret_cast<float *>(A.eval_out)[((size_t)r.x * 8 + (r.y >> 28)) * 2 + c] = out[i];
    }
}

}  // namespace b200
