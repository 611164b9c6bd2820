// dist_dev.cuh — distributional search cores (SURVEY §8a row a16; BASELINE config 5), device side.
// Restated from the reference's numba functions agents/core_distributional.py:12-124 (the agent file that should call
// them, agents/DistValueSimOnline.py, is not runnable upstream).  Arrays in the reference layout:
//   node_stats f32[M][5] = {visit, mean, reward, variance, M2}, node_dist f32[M][bins], child int32[M][7].
// The reference compiles these with fastmath (not bit-stable); parity is to 1e-5 relative.  One documented choice:
// `list(set(children))` (core_distributional.py:90-91) is taken in ascending index order.
#pragma once
#include <stdint.h>
#include "search_dev.cuh"

namespace b200 {

// core_distributional.py:12-36
__device__ inline void dist_shift(const float *dist, int bins, double x, double vmin, double vmax, float *result) {
    const double delta = (vmax - vmin) / bins, bin_shift = x / delta, fraction = bin_shift - floor(bin_shift);
    for (int b = 0; b < bins; ++b) result[b] = 0.f;
    for (int b = 0; b < bins; ++b) {
        int b_lb = (int)(b + bin_shift);
        if (b_lb >= bins) b_lb = bins - 1;
        int b_ub = (b_lb + 1 >= bins) ? bins - 1 : b_lb + 1;
        result[b_lb] = (float)__dadd_rn((double)result[b_lb], __dmul_rn((double)dist[b], 1.0 - fraction));
        result[b_ub] = (float)__dadd_rn((double)result[b_ub], __dmul_rn((double)dist[b], fraction));
    }
}

// core_distributional.py:39-45
__device__ inline double dist_mean(const float *dist, int bins, double vmin, double vmax) {
    const double delta = (vmax - vmin) / bins;
    double s = 0;
    for (int b = 0; b < bins; ++b) s = __dadd_rn(s, __dmul_rn((double)dist[b], (b + 0.5) * delta));
    return s;
}

// core_distributional.py:48-63
__device__ inline void dist_mean_variance(const float *dist, int bins, double vmin, double vmax, double &mean, double &var) {
    const double delta = (vmax - vmin) / bins;
    double m = 0, m2 = 0;
    for (int b = 0; b < bins; ++b) {
        double center = (b + 0.5) * delta, tmp = __dmul_rn(center, (double)dist[b]);
        m = __dadd_rn(m, tmp);
        m2 = __dadd_rn(m2, __dmul_rn(center, tmp));
    }
    mean = m;
    var = __dsub_rn(m2, __dmul_rn(m, m));
}

__device__ inline double dist_norm_quantile(double t) {   // agents/special.py:55-66 == special.h:26-33
    double alpha = 1.0 - 1.0 / t;
    return 10.0 * log(1.0 - log(-log(alpha) / log(2.0)) / log(22.0)) / log(41.0);
}

// core_distributional.py:66-79
__device__ inline int dist_policy(const int32_t *cn, int k, const float *node_stats, double curr_reward) {
    double n = 0;
    float s0[7], s1[7];
    for (int i = 0; i < k; ++i) {
        const float *ns = node_stats + (size_t)cn[i] * 5;
        n += (double)ns[0];
        s0[i] = (float)((double)__fadd_rn(ns[1], ns[2]) - curr_reward);
        s1[i] = (float)((double)ns[3] / ((double)ns[0] + 1e-3));
    }
    const double z = dist_norm_quantile(n);
    int best = 0; double bq = 0;
    for (int i = 0; i < k; ++i) {
        double q = (double)s0[i] + z * (double)__fsqrt_rn(s1[i]);
        if (i == 0 || q > bq) { bq = q; best = i; }
    }
    return cn[best];
}

__device__ inline int dist_unique_sorted(const int32_t *row, int32_t *out) {
    int k = 0;
    for (int a = 0; a < 7; ++a) {
        int c = row[a];
        if (c == 0) continue;
        int j = 0;
        while (j < k && out[j] != c) ++j;
        if (j == k) out[k++] = c;
    }
    for (int i = 1; i < k; ++i) { int v = out[i], j = i - 1; while (j >= 0 && out[j] > v) { out[j + 1] = out[j]; --j; } out[j + 1] = v; }
    return k;
}

// core_distributional.py:82-106 (check_low: agents/core.py:462-468, draws from the injected xorshift stream)
__device__ inline int dist_select_trace(int index, const int32_t *child, const float *node_stats, int low, int32_t *trace,
                                        int max_trace, uint32_t *rng) {
    int D = 0;
    for (;;) {
        if (D >= max_trace) return -1;
        trace[D++] = index;
        int32_t cn[7], lowl[7];
        int k = dist_unique_sorted(child + (size_t)index * 7, cn), nl = 0;
        if (k == 0) break;
        const double r = node_stats[(size_t)index * 5 + 2];
        for (int i = 0; i < k; ++i) if (node_stats[(size_t)cn[i] * 5] < (float)low) lowl[nl++] = cn[i];
        if (nl) { uint32_t s = *rng; uint32_t x = rng_next(s); *rng = s; index = lowl[x % (uint32_t)nl]; }
        else index = dist_policy(cn, k, node_stats, r);
    }
    return D;
}

// One level of backup_trace_distributional (core_distributional.py:112-124), one warp, lanes over the bins (bins <= 64): shift the
// leaf histogram d by x = r - reward (shift_distribution, :12-36), fold it into the node's running average nd, then lane 0 updates the
// node's Welford statistics ns = {visit, mean, reward, variance, M2}.  mean = dist_mean(d).
// shift_distribution is taken as a gather with the reference's bin mapping: source b goes to lb = min(int(b + bin_shift), T) with weight
// 1 - frac and to ub = min(lb + 1, T) with frac, int() truncating the DOUBLE sum.  That sum is b + s or b + s + 1 (s = int(bin_shift)):
// the second when bin_shift lies just below an integer and adding b rounds it up to that integer (DESIGN §3).  So the sources reaching
// a target tb < T lie in tb - s - 2 .. tb - s, and T also collects every source clamped onto it.  Each target adds its sources' terms
// in ascending source order, (1 - frac) before frac, each rounded to float as the scalar loop does.
__device__ inline void dist_backup_level(const float *d, int bins, double delta, double mean, double r, float *ns, float *nd, int lane) {
    const int T = bins - 1;
    // only lane 0 touches ns in memory (it rewrites it below); the others get visit and reward from its registers.  Each lane reads and
    // writes only its own bins of nd, so the levels need no other synchronisation, even when a node repeats in the trace.
    float ns0 = 0.f, ns1 = 0.f, ns2 = 0.f, ns4 = 0.f;
    if (lane == 0) { ns0 = ns[0]; ns1 = ns[1]; ns2 = ns[2]; ns4 = ns[4]; }
    ns0 = __shfl_sync(0xffffffffu, ns0, 0);
    ns2 = __shfl_sync(0xffffffffu, ns2, 0);
    const double _r = r - (double)ns2;
    const double bin_shift = _r / delta, frac = bin_shift - floor(bin_shift);
    const int s = bin_shift < (double)bins ? (int)bin_shift : bins;
    // b + bin_shift < 128 has an ulp of at most 2^-46, so it can only round up to the next integer when 1 - frac is below that: otherwise
    // every source maps to b + s: a target tb < T takes exactly tb - s - 1 (its frac) and tb - s (its 1 - frac), T takes T - s - 1 (its
    // frac) and both terms of every source from T - s on
    const bool plain = frac < 1.0 - 0x1p-40;
    for (int tb = lane; tb < bins; tb += 32) {
        float acc = 0.f;
        if (plain) {
            const int b1 = tb - s - 1, b2 = tb - s;
            if (b1 >= 0 && b1 < bins) acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b1], frac));
            if (tb < T) {
                if (b2 >= 0 && b2 < bins) acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b2], 1.0 - frac));
            } else {
                for (int b = max(b2, 0); b < bins; ++b) {
                    acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b], 1.0 - frac));
                    acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b], frac));
                }
            }
        } else {
            const int hi = tb < T ? min(tb - s, T) : T;
            for (int b = max(tb - s - 2, 0); b <= hi; ++b) {
                const double sb = __dadd_rn((double)b, bin_shift);
                const int lb = sb >= (double)T ? T : (int)sb, ub = lb + 1 >= T ? T : lb + 1;
                if (lb == tb) acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b], 1.0 - frac));
                if (ub == tb) acc = (float)__dadd_rn((double)acc, __dmul_rn((double)d[b], frac));
            }
        }
        const float num = __fadd_rn(__fmul_rn(nd[tb], ns0), acc);
        nd[tb] = (float)((double)num / ((double)ns0 + 1.0));
    }
    if (lane == 0) {
        const double x = mean + _r;
        const float n1 = __fadd_rn(ns0, 1.f);
        const double dl = x - (double)ns1;
        const float m1 = (float)((double)ns1 + dl / (double)n1);
        const double dl2 = x - (double)m1;
        const float m2 = (float)((double)ns4 + dl * dl2);
        ns[0] = n1; ns[1] = m1; ns[4] = m2;
        if (n1 > 1.f) ns[3] = (float)((double)m2 / ((double)n1 - 1.0));
    }
}

// backup_trace_distributional (core_distributional.py:109-124) for one trace, one full warp.  d: the leaf histogram in shared memory;
// node rows ns_stride floats apart in node_stats (5 in the reference layout, NSTAT_WORDS in the arena).  The engine's k_dist_backup and
// the operator b200_dist_backup_trace both run this.
__device__ inline void dist_backup_trace_warp(const float *d, int bins, double vmin, double vmax, double r, const int32_t *trace, int D,
                                              float *node_stats, int ns_stride, float *node_dist, int lane) {
    const double delta = (vmax - vmin) / bins;
    const double mean = dist_mean(d, bins, vmin, vmax);
    for (int t = 0; t < D; ++t) {
        const int idx = trace[t];
        dist_backup_level(d, bins, delta, mean, r, node_stats + (size_t)idx * ns_stride, node_dist + (size_t)idx * bins, lane);
    }
}

// ---- single-call twins (operator-level parity entry points, not the throughput path)
__global__ void k_dist_shift(const float *dist, int bins, double x, double vmin, double vmax, float *out) { dist_shift(dist, bins, x, vmin, vmax, out); }
__global__ void k_dist_mean_variance(const float *dist, int bins, double vmin, double vmax, double *out) { dist_mean_variance(dist, bins, vmin, vmax, out[0], out[1]); }
__global__ void k_dist_select(int index, const int32_t *child, const float *node_stats, int low, int32_t *trace, int max_trace, uint32_t *rng, int32_t *len) {
    *len = dist_select_trace(index, child, node_stats, low, trace, max_trace, rng);
}
__global__ void __launch_bounds__(32) k_dist_backup_trace(const int32_t *trace, int D, float *node_stats, float *node_dist, int bins, double r,
                                                           const float *dist, double vmin, double vmax) {   // one warp, bins <= 64
    __shared__ float d[64];
    for (int b = threadIdx.x; b < bins; b += 32) d[b] = dist[b];
    __syncwarp();
    dist_backup_trace_warp(d, bins, vmin, vmax, r, trace, D, node_stats, 5, node_dist, threadIdx.x);
}

}  // namespace b200
