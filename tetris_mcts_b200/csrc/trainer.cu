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
//
// Arithmetic: fp32 storage as in the reference; every contraction (forward GEMMs, weight / bias / input gradients) accumulates in fp64 and
// rounds once to fp32, so the result does not depend on a blocking order and sits within the reference's own fp32 rounding noise
// (tests: rtol 1e-5 against goldens recorded from the reference's own Model_VV.train on torch CPU).  Convolutions are lowered to
// GEMMs through explicit im2col buffers in HBM (the PyTorch [co][ci][ky][kx] weight layout is used as it lies: k = ci*9 + ky*3 + kx).
// No atomics: every reduction has a fixed order, training is bit-reproducible run to run.
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200_tetris_mcts.h"

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

// out[i] = float(sum_z part[z][i] (+ bias[i % N] when bias)), optional ReLU; also used to finish single-split GEMMs
__global__ void k_finish(const double *__restrict__ part, int splits, size_t MN, int N, const float *__restrict__ bias, int relu, float *__restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < MN; i += (size_t)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int z = 0; z < splits; ++z) s += part[(size_t)z * MN + i];
        float v = (float)s;
        if (bias) v = v + bias[i % N];
        if (relu) v = fmaxf(v, 0.f);
        out[i] = v;
    }
}

// column sums: out[n] = float(sum_m X[m][n]) in fp64, one CTA per 32 columns, fixed order (rows strided over 8 warps, then a tree)
__global__ void __launch_bounds__(256) k_colsum(const float *__restrict__ X, int M, int N, float *__restrict__ out) {
    __shared__ double s[8][32];
    const int n = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
    double a = 0.0;
    if (n < N) for (int m = w; m < M; m += 8) a += (double)X[(size_t)m * N + n];
    s[w][threadIdx.x & 31] = a;
    __syncthreads();
    if (w == 0 && n < N) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += s[i][threadIdx.x & 31];
        out[n] = (float)t;
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
// One thread per sample: z = h . Wo^T + bo (fp64 accumulate), s = sigmoid(z), pred = s * ub + lb (model_vv.py:48-52), GaussianLL
// (model_vv.py:94-101) with the target variance clamped at 0.1 (:140), weight applied when `weighted` (:145-149); and the gradient of
// mean(w * logl) with respect to z (the two pre-sigmoid outputs).
__global__ void k_head(const float *__restrict__ h, const float *__restrict__ Wo, const float *__restrict__ bo, const float *__restrict__ ub,
                       const float *__restrict__ lb, const float *__restrict__ value, const float *__restrict__ variance, const float *__restrict__ weight,
                       int B, int weighted, float *__restrict__ pred, float *__restrict__ lossv, float *__restrict__ dz) {
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
    const float gl = w / (float)B;                                  // d mean(w * logl) / d logl_b
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

inline int nblk(size_t n, int t = 256) { size_t b = (n + t - 1) / t; return (int)(b < 1 ? 1 : (b > 132 * 16 ? 132 * 16 : b)); }

}  // namespace

struct b200_trainer {
    int device = 0, max_batch = 0;
    cudaStream_t stream = nullptr;
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
    double *part; size_t part_elems = 0;
};

namespace {

template <typename T> int talloc(b200_trainer *t, T **p, size_t n) {
    void *q = nullptr;
    if (cudaMalloc(&q, (n ? n : 1) * sizeof(T)) != cudaSuccess) return tfail(B200_ERR_CUDA, "cudaMalloc failed (trainer, " + std::to_string(n * sizeof(T)) + " B)");
    t->allocs.push_back(q);
    *p = (T *)q;
    return 0;
}

// C = op(A) op(B) with fp64 accumulation, optional bias / ReLU; split-k for long reductions (fixed order)
template <bool TA, bool TB>
int gemm(b200_trainer *t, const float *A, const float *B, float *C, int M, int N, int K, const float *bias, int relu) {
    int splits = 1;
    const int tiles = ((M + 63) / 64) * ((N + 63) / 64);
    if (K >= 4096 && tiles < 132 * 2) { splits = (132 * 4 + tiles - 1) / tiles; if (splits > (K + 511) / 512) splits = (K + 511) / 512; }
    int kps = ((K + splits - 1) / splits + 15) / 16 * 16;
    splits = (K + kps - 1) / kps;
    dim3 grid((N + 63) / 64, (M + 63) / 64, splits);
    if (splits == 1) {
        k_gemm<TA, TB><<<grid, 256, 0, t->stream>>>(A, B, nullptr, M, N, K, kps, C, bias, relu);
        return 0;
    }
    if ((size_t)splits * M * N > t->part_elems) return tfail(B200_ERR_BAD_ARG, "trainer: partial-sum buffer too small");
    k_gemm<TA, TB><<<grid, 256, 0, t->stream>>>(A, B, t->part, M, N, K, kps, nullptr, nullptr, 0);
    k_finish<<<nblk((size_t)M * N), 256, 0, t->stream>>>(t->part, splits, (size_t)M * N, N, bias, relu, C);
    return 0;
}

int forward(b200_trainer *t, int B) {
    float *W = t->w;
    int rc = 0;
    k_im2col<<<nblk((size_t)B * 144 * 9), 256, 0, t->stream>>>(t->x0, B, 20, 10, 1, t->col1);
    rc |= gemm<false, true>(t, t->col1, W + O_C1W, t->a1, B * 144, 32, 9, W + O_C1B, 1);          // model_vv.py:32-33
    k_im2col<<<nblk((size_t)B * 96 * 288), 256, 0, t->stream>>>(t->a1, B, 18, 8, 32, t->col2);
    rc |= gemm<false, true>(t, t->col2, W + O_C2W, t->a2, B * 96, 32, 288, W + O_C2B, 1);          // :34-35
    k_im2col<<<nblk((size_t)B * 56 * 288), 256, 0, t->stream>>>(t->a2, B, 16, 6, 32, t->col3);
    rc |= gemm<false, true>(t, t->col3, W + O_C3W, t->a3, B * 56, 32, 288, W + O_C3B, 1);          // :36-37
    k_nhwc_to_flat<<<nblk((size_t)B * 1792), 256, 0, t->stream>>>(t->a3, B, t->flat);              // :38 nn.Flatten on NCHW
    rc |= gemm<false, true>(t, t->flat, W + O_F1W, t->h, B, 256, 1792, W + O_F1B, 1);              // :39-40
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
    k_head<<<(B + 127) / 128, 128, 0, t->stream>>>(t->h, W + O_FOW, W + O_FOB, W + O_UB, W + O_LB, t->value, t->variance, t->weight, B, weighted,
                                                   t->pred, t->lossv, want_grad ? t->dz : nullptr);
    k_std_mean<<<1, 256, 0, t->stream>>>(t->lossv, B, t->d_lossstat);
    double h2[2];
    TCK(cudaMemcpyAsync(h2, t->d_lossstat, 16, cudaMemcpyDeviceToHost, t->stream));
    TCK(cudaStreamSynchronize(t->stream));
    if (loss) *loss = h2[0];
    if (loss_std) *loss_std = h2[1];
    return 0;
}

int backward(b200_trainer *t, int B) {
    float *W = t->w, *G = t->grad;
    int rc = 0;
    // fc_out: dWo[j][k] = sum_b dz[b][j] h[b][k]; dbo[j] = sum_b dz[b][j]
    rc |= gemm<true, false>(t, t->dz, t->h, G + O_FOW, 2, 256, B, nullptr, 0);
    k_colsum<<<1, 256, 0, t->stream>>>(t->dz, B, 2, G + O_FOB);
    k_dh<<<nblk((size_t)B * 256), 256, 0, t->stream>>>(t->dz, W + O_FOW, t->h, B, t->dh);
    // fc1: dW1[n][k] = sum_b dh[b][n] flat[b][k]; db1; dflat = dh . W1
    rc |= gemm<true, false>(t, t->dh, t->flat, G + O_F1W, 256, 1792, B, nullptr, 0);
    k_colsum<<<8, 256, 0, t->stream>>>(t->dh, B, 256, G + O_F1B);
    rc |= gemm<false, false>(t, t->dh, W + O_F1W, t->dflat, B, 1792, 256, nullptr, 0);
    k_flat_to_nhwc_relu<<<nblk((size_t)B * 1792), 256, 0, t->stream>>>(t->dflat, t->flat, B, t->dc3);   // ReLU after conv3 (act3)
    // conv3
    rc |= gemm<true, false>(t, t->dc3, t->col3, G + O_C3W, 32, 288, B * 56, nullptr, 0);
    k_colsum<<<1, 256, 0, t->stream>>>(t->dc3, B * 56, 32, G + O_C3B);
    rc |= gemm<false, false>(t, t->dc3, W + O_C3W, t->dcol3, B * 56, 288, 32, nullptr, 0);
    k_col2im_relu<<<nblk((size_t)B * 96 * 32), 256, 0, t->stream>>>(t->dcol3, t->a2, B, 16, 6, 32, t->da2);
    // conv2
    rc |= gemm<true, false>(t, t->da2, t->col2, G + O_C2W, 32, 288, B * 96, nullptr, 0);
    k_colsum<<<1, 256, 0, t->stream>>>(t->da2, B * 96, 32, G + O_C2B);
    rc |= gemm<false, false>(t, t->da2, W + O_C2W, t->dcol2, B * 96, 288, 32, nullptr, 0);
    k_col2im_relu<<<nblk((size_t)B * 144 * 32), 256, 0, t->stream>>>(t->dcol2, t->a1, B, 18, 8, 32, t->da1);
    // conv1 (no input gradient needed)
    rc |= gemm<true, false>(t, t->da1, t->col1, G + O_C1W, 32, 9, B * 144, nullptr, 0);
    k_colsum<<<1, 256, 0, t->stream>>>(t->da1, B * 144, 32, G + O_C1B);
    return rc;
}

}  // namespace

extern "C" const char *b200_trainer_last_error(void) { return g_terr.c_str(); }

extern "C" int b200_trainer_destroy(b200_trainer *t) {
    if (!t) return B200_OK;
    if (t->stream) cudaStreamSynchronize(t->stream);
    for (void *p : t->allocs) cudaFree(p);
    if (t->stream) cudaStreamDestroy(t->stream);
    delete t;
    return B200_OK;
}

extern "C" int b200_trainer_create(int device, const float *weights, int max_batch, b200_trainer **out) {
    if (!weights || !out || max_batch < 1 || max_batch > 65536) return tfail(B200_ERR_BAD_ARG, "trainer: bad argument (1 <= max_batch <= 65536)");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return tfail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TCK(cudaSetDevice(device));
    b200_trainer *t = new b200_trainer();
    struct Guard { b200_trainer *t; ~Guard() { if (t) b200_trainer_destroy(t); } } guard{t};
    t->device = device; t->max_batch = max_batch;
    TCK(cudaStreamCreateWithFlags(&t->stream, cudaStreamNonBlocking));
    const size_t B = (size_t)max_batch;
    int rc = 0;
    rc |= talloc(t, &t->w, N_ALL); rc |= talloc(t, &t->grad, N_TRAIN); rc |= talloc(t, &t->m, N_TRAIN); rc |= talloc(t, &t->v, N_TRAIN);
    rc |= talloc(t, &t->d_toff, N_TENSORS + 1); rc |= talloc(t, &t->d_sumsq, N_TENSORS); rc |= talloc(t, &t->d_lossstat, 2);
    rc |= talloc(t, &t->d_states, B * 200); rc |= talloc(t, &t->d_idx, B);
    rc |= talloc(t, &t->x0, B * 200); rc |= talloc(t, &t->value, B); rc |= talloc(t, &t->variance, B); rc |= talloc(t, &t->weight, B);
    rc |= talloc(t, &t->col1, B * 144 * 9); rc |= talloc(t, &t->a1, B * 144 * 32); rc |= talloc(t, &t->col2, B * 96 * 288); rc |= talloc(t, &t->a2, B * 96 * 32);
    rc |= talloc(t, &t->col3, B * 56 * 288); rc |= talloc(t, &t->a3, B * 56 * 32); rc |= talloc(t, &t->flat, B * 1792); rc |= talloc(t, &t->h, B * 256);
    rc |= talloc(t, &t->pred, B * 2); rc |= talloc(t, &t->lossv, B); rc |= talloc(t, &t->dz, B * 2);
    rc |= talloc(t, &t->dh, B * 256); rc |= talloc(t, &t->dflat, B * 1792); rc |= talloc(t, &t->dc3, B * 56 * 32); rc |= talloc(t, &t->dcol3, B * 56 * 288);
    rc |= talloc(t, &t->da2, B * 96 * 32); rc |= talloc(t, &t->dcol2, B * 96 * 288); rc |= talloc(t, &t->da1, B * 144 * 32);
    // split-k partial sums (fp64): only the weight-gradient products are split; the largest is fc1 (256 x 1792) with <= 8 k ranges
    t->part_elems = (size_t)8 * 256 * 1792;
    rc |= talloc(t, &t->part, t->part_elems);
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
