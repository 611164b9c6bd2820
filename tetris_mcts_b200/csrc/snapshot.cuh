// snapshot.cuh — device side of b200_engine_save / b200_engine_load: each game's arena packed to the words a later call can read before it
// writes them, and scattered back into a freshly created (zeroed) engine.  One CTA per game, in the style of k_gc.
//
// Packed game (u32 words; RW = ROW_WORDS, plus NSTAT_WORDS + dist_bins in MODE_DIST):
//   [0, SNAP_HDR)   g, n_nfree, n_ofree, root, episode, status, srng, trace_len, leaf_kind, pending, resume_a, node entries, obs entries,
//                   cur[REC_WORDS]
//   nfree[n_nfree], ofree[n_ofree]                   the free lists as they are (popped from the back)
//   rec[M][REC_WORDS]                                every node slot: a freed slot's record is what stale_pop erases by, and records are
//                                                    allocated without zeroing
//   row[M - n_nfree][RW]                             live node slots (slot 0 included) in ascending order
//   row word 15 of nfree[j], j < n_nfree             k_gc zeroes a freed row except o[7]
//   {stat[4], key[12]}[M - n_ofree]                  live observation slots in ascending order (freed ones are zero)
//   {hash32, index}[node entries], [obs entries]     the tables' entry lists, re-inserted with tab_home / tab_next as k_gc does
//   trace[trace_len]                                 the last trace (b200_export_game reads it)
//   checksum (2 words)                               snap_checksum of everything before it
#pragma once
#include "kernels.cuh"

namespace b200 {

constexpr int SNAP_HDR = 13 + REC_WORDS;

__host__ __device__ inline int snap_row_words(int mode, int bins) { return ROW_WORDS + (mode == MODE_DIST ? NSTAT_WORDS + bins : 0); }

// packed size in words of a game with these counts
__host__ __device__ inline long long snap_game_words(int M, int rw, int nn, int no, int ne_n, int ne_o, int tl) {
    return (long long)SNAP_HDR + nn + no + (long long)M * REC_WORDS + (long long)(M - nn) * rw + nn + (long long)(M - no) * (4 + KEY_WORDS) +
           2LL * (ne_n + ne_o) + tl + 2;
}

__device__ __forceinline__ uint64_t snap_mix(uint64_t x) {   // splitmix64's finaliser
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// sum over i of mix(i, w[i]): a flipped bit anywhere changes one term.  The whole block calls it; every thread gets the sum.
__device__ __forceinline__ uint64_t snap_checksum(const uint32_t *w, long long n, unsigned long long *s_sum) {
    uint64_t part = 0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) part += snap_mix(((uint64_t)i << 32) ^ w[i]);
    __syncthreads();
    if (threadIdx.x == 0) *s_sum = 0ull;
    __syncthreads();
    atomicAdd(s_sum, (unsigned long long)part);
    __syncthreads();
    const uint64_t tot = *s_sum;
    __syncthreads();
    return tot;
}

// per game: its packed size (words) and its two tables' entry counts
__global__ void k_snap_count(Arena A, long long *words, int32_t *entries) {
    const int g = blockIdx.x;
    __shared__ int s_n[2];
    if (threadIdx.x < 2) s_n[threadIdx.x] = 0;
    __syncthreads();
    const uint2 *ntab = A.ntab + (size_t)g * A.H, *otab = A.otab + (size_t)g * A.H;
    int cn = 0, co = 0;
    for (int p = threadIdx.x; p < A.H; p += blockDim.x) {
        const uint32_t yn = ntab[p].y, yo = otab[p].y;
        cn += yn != 0u && yn != 0xffffffffu;
        co += yo != 0u && yo != 0xffffffffu;
    }
    atomicAdd(&s_n[0], cn); atomicAdd(&s_n[1], co);
    __syncthreads();
    if (threadIdx.x == 0) {
        int tl = A.trace_len[g];
        tl = tl < 0 ? 0 : (tl > A.trace_max ? A.trace_max : tl);
        entries[2 * g] = s_n[0]; entries[2 * g + 1] = s_n[1];
        words[g] = snap_game_words(A.M, snap_row_words(A.mode, A.dist_bins), A.n_nfree[g], A.n_ofree[g], s_n[0], s_n[1], tl);
    }
}

// the live slots of one game in ascending order -> list[0 .. n): mark[i] != 0 = slot i is free.  Returns n (every thread).
__device__ __forceinline__ int snap_live_list(const uint8_t *mark, int M, int32_t *list, int *s_warp) {
    int n = 0;
    for (int base = 0; base < M; base += GC_THREADS) {
        const int i = base + threadIdx.x;
        const int f = i < M && !mark[i];
        int tot;
        const int r = block_excl_scan(f, s_warp, tot);
        if (f) list[n + r] = i;
        n += tot;
    }
    __syncthreads();
    return n;
}

// marks of the free slots (nmark / omark of this CTA's collection scratch); returns how many distinct slots in [1, M) the lists name
__device__ __forceinline__ int snap_free_marks(const int32_t *nfree, int nn, const int32_t *ofree, int no, int M, uint8_t *nmark, uint8_t *omark,
                                               int *s_cnt) {
    for (int i = threadIdx.x; i < M; i += GC_THREADS) { nmark[i] = 0; omark[i] = 0; }
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int j = threadIdx.x; j < nn; j += GC_THREADS) { const int i = nfree[j]; if (i >= 1 && i < M && test_and_set_mark(nmark, i)) ++c; }
    for (int j = threadIdx.x; j < no; j += GC_THREADS) { const int i = ofree[j]; if (i >= 1 && i < M && test_and_set_mark(omark, i)) ++c; }
    atomicAdd(s_cnt, c);
    __syncthreads();
    const int tot = *s_cnt;
    __syncthreads();
    return tot;
}

// games [g0, g1) into out; game g at out + off[g] - base.  Grid: at most gc_pool_main CTAs (each uses one collection scratch set).
__global__ void __launch_bounds__(GC_THREADS) k_snap_pack(Arena A, int g0, int g1, const long long *off, long long base, const int32_t *entries,
                                                          uint32_t *out) {
    __shared__ int s_warp[GC_THREADS / 32];
    __shared__ int s_n;
    __shared__ unsigned long long s_sum;
    const int t = threadIdx.x, M = A.M, H = A.H;
    const int rw = snap_row_words(A.mode, A.dist_bins), bins = A.dist_bins;
    uint8_t *nmark = A.nmark + (size_t)blockIdx.x * M, *omark = A.omark + (size_t)blockIdx.x * M;
    int32_t *nlist = A.gc_queue + (size_t)blockIdx.x * 2 * M, *olist = nlist + M;
    for (int g = g0 + blockIdx.x; g < g1; g += gridDim.x) {
        uint32_t *o = out + (off[g] - base);
        const int nn = A.n_nfree[g], no = A.n_ofree[g];
        const int32_t *nfree = A.nfree + (size_t)g * M, *ofree = A.ofree + (size_t)g * M;
        snap_free_marks(nfree, nn, ofree, no, M, nmark, omark, &s_n);
        const int nl = snap_live_list(nmark, M, nlist, s_warp), ol = snap_live_list(omark, M, olist, s_warp);
        int tl = A.trace_len[g];
        tl = tl < 0 ? 0 : (tl > A.trace_max ? A.trace_max : tl);
        const int ne_n = entries[2 * g], ne_o = entries[2 * g + 1];
        if (t == 0) {
            o[0] = g; o[1] = nn; o[2] = no; o[3] = A.root[g]; o[4] = A.episode[g]; o[5] = A.status[g]; o[6] = A.srng[g];
            o[7] = tl; o[8] = A.leaf_kind[g]; o[9] = A.pending[g]; o[10] = A.resume_a[g]; o[11] = ne_n; o[12] = ne_o;
        }
        if (t < REC_WORDS) o[13 + t] = A.cur[(size_t)g * REC_WORDS + t];
        long long p = SNAP_HDR;
        for (int j = t; j < nn; j += GC_THREADS) o[p + j] = nfree[j];
        p += nn;
        for (int j = t; j < no; j += GC_THREADS) o[p + j] = ofree[j];
        p += no;
        const uint32_t *recb = A.rec + (size_t)g * M * REC_WORDS;
        for (long long k = t; k < (long long)M * REC_WORDS; k += GC_THREADS) o[p + k] = recb[k];
        p += (long long)M * REC_WORDS;
        const int32_t *rowb = A.row + (size_t)g * M * ROW_WORDS;
        const float *nsb = A.nstat ? A.nstat + (size_t)g * M * NSTAT_WORDS : nullptr, *ndb = A.nstat ? A.ndist + (size_t)g * M * bins : nullptr;
        for (long long k = t; k < (long long)nl * rw; k += GC_THREADS) {
            const int i = nlist[k / rw], w = (int)(k % rw);
            o[p + k] = w < ROW_WORDS ? (uint32_t)rowb[(size_t)i * ROW_WORDS + w]
                     : (w < ROW_WORDS + NSTAT_WORDS ? __float_as_uint(nsb[(size_t)i * NSTAT_WORDS + w - ROW_WORDS])
                                                    : __float_as_uint(ndb[(size_t)i * bins + w - ROW_WORDS - NSTAT_WORDS]));
        }
        p += (long long)nl * rw;
        for (int j = t; j < nn; j += GC_THREADS) o[p + j] = rowb[(size_t)nfree[j] * ROW_WORDS + 15];
        p += nn;
        const uint32_t *statb = reinterpret_cast<const uint32_t *>(A.stat + (size_t)g * M), *keyb = A.key + (size_t)g * M * KEY_WORDS;
        for (long long k = t; k < (long long)ol * 16; k += GC_THREADS) {
            const int i = olist[k >> 4], w = (int)(k & 15);
            o[p + k] = w < 4 ? statb[(size_t)i * 4 + w] : keyb[(size_t)i * KEY_WORDS + w - 4];
        }
        p += (long long)ol * 16;
        for (int tb = 0; tb < 2; ++tb) {          // entry lists in table order (keys are unique: any insertion order finds the same index)
            const uint2 *tab = (tb ? A.otab : A.ntab) + (size_t)g * H;
            int c = 0;
            for (int b = 0; b < H; b += GC_THREADS) {
                const int q = b + t;
                const uint2 e = q < H ? tab[q] : make_uint2(0u, 0u);
                const int f = e.y != 0u && e.y != 0xffffffffu;
                int tot;
                const int r = block_excl_scan(f, s_warp, tot);
                if (f) { o[p + 2 * (c + r)] = e.x; o[p + 2 * (c + r) + 1] = e.y; }
                c += tot;
            }
            p += 2LL * (tb ? ne_o : ne_n);
        }
        const int32_t *tr = A.trace + (size_t)g * A.trace_max;
        for (int j = t; j < tl; j += GC_THREADS) o[p + j] = tr[j];
        p += tl;
        __syncthreads();
        const uint64_t cs = snap_checksum(o, p, &s_sum);
        if (t == 0) { o[p] = (uint32_t)cs; o[p + 1] = (uint32_t)(cs >> 32); }
        __syncthreads();
    }
}

// The inverse of k_snap_pack into a freshly created engine (rows, statistics, keys, tables zero).  A game whose checksum, header or indices
// do not hold is left untouched and reported: *err = min over such games of game << 8 | reason (one 64-bit atomicMin, so the reason is the
// first game's own; ~0 = none), reason 1 checksum, 2 header / size / per-game word, 3 free lists, 4 an index or key cell out of range.
__global__ void __launch_bounds__(GC_THREADS) k_snap_unpack(Arena A, int g0, int g1, const long long *off, long long base, const uint32_t *in,
                                                            unsigned long long *err) {
    __shared__ int s_warp[GC_THREADS / 32];
    __shared__ int s_n, s_bad;
    __shared__ unsigned long long s_sum;
    const int t = threadIdx.x, M = A.M, H = A.H;
    const int rw = snap_row_words(A.mode, A.dist_bins), bins = A.dist_bins;
    uint8_t *nmark = A.nmark + (size_t)blockIdx.x * M, *omark = A.omark + (size_t)blockIdx.x * M;
    int32_t *nlist = A.gc_queue + (size_t)blockIdx.x * 2 * M, *olist = nlist + M;
    for (int g = g0 + blockIdx.x; g < g1; g += gridDim.x) {
        const uint32_t *w = in + (off[g] - base);
        const long long size = off[g + 1] - off[g];
        if (t == 0) s_bad = 0;
        __syncthreads();
        // the checksum first: nothing of a corrupted game is interpreted
        const uint64_t cs = snap_checksum(w, size - 2, &s_sum);
        if (t == 0 && (uint32_t)cs != w[size - 2]) s_bad = 1;
        if (t == 0 && (uint32_t)(cs >> 32) != w[size - 1]) s_bad = 1;
        __syncthreads();
        const int nn = (int)w[1], no = (int)w[2], tl = (int)w[7], ne_n = (int)w[11], ne_o = (int)w[12];
        if (t == 0 && !s_bad) {
            const bool ok = (int)w[0] == g && nn >= 0 && nn < M && no >= 0 && no < M && tl >= 0 && tl <= A.trace_max && ne_n >= 0 && ne_n <= M &&
                            ne_o >= 0 && ne_o <= M && (int)w[3] >= 0 && (int)w[3] < M && w[5] <= (uint32_t)ST_RESET_DONE &&
                            w[8] <= (uint32_t)LEAF_DONE && w[9] <= (uint32_t)PEND_ROOT && w[10] <= 7u &&
                            size == snap_game_words(M, rw, nn, no, ne_n, ne_o, tl);
            if (!ok) s_bad = 2;
        }
        __syncthreads();
        if (s_bad) { if (t == 0) atomicMin(err, (unsigned long long)g << 8 | (unsigned)s_bad); __syncthreads(); continue; }
        const int32_t *nfree = reinterpret_cast<const int32_t *>(w + SNAP_HDR), *ofree = nfree + nn;
        if (snap_free_marks(nfree, nn, ofree, no, M, nmark, omark, &s_n) != nn + no) {   // an index out of [1, M) or named twice
            if (t == 0) atomicMin(err, (unsigned long long)g << 8 | 3u);
            __syncthreads();
            continue;
        }
        const int nl = snap_live_list(nmark, M, nlist, s_warp), ol = snap_live_list(omark, M, olist, s_warp);
        const long long p_rec = SNAP_HDR + nn + no, p_row = p_rec + (long long)M * REC_WORDS, p_w15 = p_row + (long long)nl * rw;
        const long long p_obs = p_w15 + nn, p_tab = p_obs + (long long)ol * 16, p_tr = p_tab + 2LL * (ne_n + ne_o);
        // every index a later kernel follows: the rows' child ids, observation ids and de-duplicated child lists (node ids under
        // LINK_NODE_MASK), the free rows' o[7], the table entries, the trace, and the cells of the falling piece in the live keys (k_gc and
        // k_collect_samples write them as byte offsets into a 212-byte replay row; obskey gives four cells < 200)
        int bad = 0;
        for (long long k = t; k < (long long)nl * rw; k += GC_THREADS) {
            const int wd = (int)(k % rw);
            const uint32_t v = w[p_row + k];
            if ((wd < 7 || (wd >= 8 && wd < 16)) && v >= (uint32_t)M) bad = 1;
            if (wd >= 24 && wd < 31 && (v & LINK_NODE_MASK) >= (uint32_t)M) bad = 1;
        }
        for (int j = t; j < ol; j += GC_THREADS) {
            const uint32_t cells = w[p_obs + (long long)j * 16 + 4 + 10];
            for (int q = 0; q < 4; ++q) bad |= ((cells >> (8 * q)) & 0xffu) >= 200u;
        }
        for (int j = t; j < nn; j += GC_THREADS) bad |= w[p_w15 + j] >= (uint32_t)M;
        for (int j = t; j < ne_n + ne_o; j += GC_THREADS) { const uint32_t y = w[p_tab + 2 * j + 1]; bad |= y == 0u || y >= (uint32_t)M; }
        for (int j = t; j < tl; j += GC_THREADS) bad |= w[p_tr + j] >= (uint32_t)M;
        if (bad) atomicOr(&s_bad, 4);
        __syncthreads();
        if (s_bad) { if (t == 0) atomicMin(err, (unsigned long long)g << 8 | 4u); __syncthreads(); continue; }
        if (t == 0) {
            A.n_nfree[g] = nn; A.n_ofree[g] = no; A.root[g] = (int)w[3]; A.episode[g] = (int)w[4]; A.status[g] = (int)w[5]; A.srng[g] = w[6];
            A.trace_len[g] = tl; A.leaf_kind[g] = (int)w[8]; A.pending[g] = (int)w[9]; A.resume_a[g] = (int)w[10];
        }
        if (t < REC_WORDS) A.cur[(size_t)g * REC_WORDS + t] = w[13 + t];
        int32_t *dn = A.nfree + (size_t)g * M, *dof = A.ofree + (size_t)g * M;
        for (int j = t; j < nn; j += GC_THREADS) dn[j] = nfree[j];
        for (int j = t; j < no; j += GC_THREADS) dof[j] = ofree[j];
        uint32_t *recb = A.rec + (size_t)g * M * REC_WORDS;
        for (long long k = t; k < (long long)M * REC_WORDS; k += GC_THREADS) recb[k] = w[p_rec + k];
        int32_t *rowb = A.row + (size_t)g * M * ROW_WORDS;
        float *nsb = A.nstat ? A.nstat + (size_t)g * M * NSTAT_WORDS : nullptr, *ndb = A.nstat ? A.ndist + (size_t)g * M * bins : nullptr;
        for (long long k = t; k < (long long)nl * rw; k += GC_THREADS) {
            const int i = nlist[k / rw], wd = (int)(k % rw);
            const uint32_t v = w[p_row + k];
            if (wd < ROW_WORDS) rowb[(size_t)i * ROW_WORDS + wd] = (int32_t)v;
            else if (wd < ROW_WORDS + NSTAT_WORDS) nsb[(size_t)i * NSTAT_WORDS + wd - ROW_WORDS] = __uint_as_float(v);
            else ndb[(size_t)i * bins + wd - ROW_WORDS - NSTAT_WORDS] = __uint_as_float(v);
        }
        for (int j = t; j < nn; j += GC_THREADS) rowb[(size_t)nfree[j] * ROW_WORDS + 15] = (int32_t)w[p_w15 + j];
        uint32_t *statb = reinterpret_cast<uint32_t *>(A.stat + (size_t)g * M), *keyb = A.key + (size_t)g * M * KEY_WORDS;
        for (long long k = t; k < (long long)ol * 16; k += GC_THREADS) {
            const int i = olist[k >> 4], wd = (int)(k & 15);
            if (wd < 4) statb[(size_t)i * 4 + wd] = w[p_obs + k];
            else keyb[(size_t)i * KEY_WORDS + wd - 4] = w[p_obs + k];
        }
        for (int tb = 0; tb < 2; ++tb) {          // re-insert as k_gc rebuilds its tables: keys are unique, so the claim order is free
            uint2 *tab = (tb ? A.otab : A.ntab) + (size_t)g * H;
            const uint32_t *e = w + p_tab + (tb ? 2LL * ne_n : 0);
            const int cnt = tb ? ne_o : ne_n;
            for (int j = t; j < cnt; j += GC_THREADS) {
                uint32_t q = tab_home(e[2 * j], H);
                while (atomicCAS(&tab[q].y, 0u, e[2 * j + 1]) != 0u) q = tab_next(q, H);
                tab[q].x = e[2 * j];
            }
        }
        int32_t *tr = A.trace + (size_t)g * A.trace_max;
        for (int j = t; j < tl; j += GC_THREADS) tr[j] = (int32_t)w[p_tr + j];
        __syncthreads();
    }
}

}  // namespace b200
