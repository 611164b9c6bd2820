// capi.cu — host side of libb200_tetris_mcts.so: the C-ABI declared in include/b200_tetris_mcts.h.
// One engine = one CUDA stream + the per-game arenas in HBM.  No CPU compute path exists in this file: every
// entry point either launches kernels or moves bytes.
#include <cuda_runtime.h>
#include <unistd.h>
#include <array>
#include <cerrno>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/b200_tetris_mcts.h"
#include "kernels.cuh"
#include "valuenet_simt.cuh"
#include "dist_dev.cuh"
#include "distnet_simt.cuh"
#include "replay_policy.cuh"
#include "valuenet_tc.cuh"
#include "distnet_tc.cuh"
#include "ext_eval.cuh"
#include "snapshot.cuh"

using namespace b200;

static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }
#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t _e = (call);                                                                      \
        if (_e != cudaSuccess)                                                                        \
            return fail(B200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_e));           \
    } while (0)

extern "C" const char *b200_last_error(void) { return g_err.c_str(); }
extern "C" int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

enum { PH_SELECT = 0, PH_CONV, PH_FC, PH_BACKUP, PH_ROLLOUT, PH_SYNTH, PH_MISC, PH_GC, PH_N = 8 };

struct b200_engine {
    b200_config cfg;
    Arena A;
    cudaStream_t stream = nullptr; bool own_stream = true;   // own_stream false: the caller's stream (b200_engine_set_stream), never destroyed here
    std::vector<void *> allocs;
    uint32_t *d_default_rec = nullptr;
    float *d_stats = nullptr; int32_t *d_action = nullptr;
    unsigned long long *d_game_stats = nullptr;
    // network
    bool have_weights = false;
    float *d_wraw = nullptr;
    NetWeights W{};
    float *d_act3 = nullptr; size_t act3_rows = 0;
    void *tc_state = nullptr; void *dn_tc_state = nullptr;
    bool have_dist_weights = false; float *d_dnw = nullptr; DistNetWeights DW{}; float *d_dn_act = nullptr; size_t dn_rows = 0;
    std::vector<float> h_w, h_dnw;   // the weights as the caller passed them (state_dict order): what b200_engine_save writes
    int dn_atoms = 0;
    int n_sm = 132;
    // timing
    bool timing = false;
    std::vector<cudaEvent_t> ev; size_t ev_used = 0;
    std::vector<int> ev_phase;
    float phase_ms[PH_N] = {0}; uint64_t phase_launches[PH_N] = {0};
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    // sampling
    uint8_t *d_samples = nullptr; int sample_cap = 0; int32_t *d_sample_count = nullptr;
    // replay-memory policy (agent.cpp:619-775)
    ReplayPolicy rp; uint8_t *d_rp_tmp = nullptr, *d_rp_keep = nullptr; float *d_rp_vis = nullptr; int32_t *d_rp_kept = nullptr; int replay_alloc = 0;
    // one simulation step captured as a CUDA graph (replayed when phase timing is off: ~7 launches + 1 memset per step, 500 steps/move)
    int gc_headroom = 0;           // b200_set_gc_headroom: collect between moves every game with fewer free slots than this
    int4 *d_pc = nullptr; int32_t *d_pc_var = nullptr, *d_pc_len = nullptr; uint4 *d_pc_sib = nullptr; int4 *d_pc_own = nullptr;   // path cache (b200_set_path_cache): allocated at the first switch-on, A.pc == nullptr while off
    // deep lane (b200_set_deep_lane): the games with the longest traces select / collect / resume on a second stream (kernels.cuh: k_classify)
    int deep_cap = 0; cudaStream_t stream1 = nullptr; cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int32_t *d_glist0 = nullptr, *d_glist1 = nullptr, *d_nlist = nullptr, *d_nreq_deep = nullptr, *d_gc_list_deep = nullptr; uint2 *d_req_deep = nullptr;
    int gc_pool_main = 0;          // collection scratch sets of the main k_gc launch; DEEP_GC_BLOCKS more follow for the deep lane's
    cudaGraphExec_t step_exec = nullptr; bool step_graph_failed = false;
    uint64_t step_launches[PH_N] = {0};
    // caller-supplied evaluator (B200_EVAL_EXTERNAL): k_ext_order's marks and ordered rows ({game, leaf} per game with
    // B200_EVAL_EXTERNAL_GAME); ext_open between b200_ext_step_begin and _end
    int32_t *d_ext_mark = nullptr, *d_ext_n = nullptr; uint2 *d_ext_rows = nullptr;
    bool ext_open = false; int32_t ext_rows = 0;
};

static bool ext_game_kind(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_EXTERNAL_GAME; }
static bool ext_kind(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_EXTERNAL || ext_game_kind(e); }
// the calls an external engine has no use for (it has no network of its own, and its steps need the caller's outputs)
static int ext_refuse(const b200_engine *e, const char *fn) {
    if (ext_game_kind(e))
        return fail(B200_ERR_BAD_ARG, std::string(fn) + ": eval_kind external_game has no built-in evaluator; drive the search with "
                                      "b200_ext_step_begin / b200_ext_step_end");
    return fail(B200_ERR_BAD_ARG, std::string(fn) + ": eval_kind external has no built-in network; drive the search with "
                                  "b200_ext_step_begin / b200_ext_step_end");
}
// the calls that change the trees, the games or the engine's stream, while a step is open between b200_ext_step_begin and _end
static int step_open(const b200_engine *e, const char *fn) {
    return fail(B200_ERR_BAD_ARG, std::string(fn) + ": a simulation step is open; finish it with b200_ext_step_end first");
}
#define REFUSE_IF_EXT(e, fn) do { if (ext_kind(e)) return ext_refuse(e, fn); } while (0)
#define REFUSE_IF_OPEN(e, fn) do { if ((e)->ext_open) return step_open(e, fn); } while (0)

// kernel arguments of the captured step changed (weights, replay memory, ...): capture again at the next run_sims
static void drop_step_graph(b200_engine *e) {
    if (e->step_exec) { cudaStreamSynchronize(e->stream); cudaGraphExecDestroy(e->step_exec); e->step_exec = nullptr; }
    e->step_graph_failed = false;
}

constexpr int DEEP_GC_BLOCKS = 8;

// k_backup's per-warp bitmap of the trace's observations (path cache on): max_nodes bits, four warps per CTA
static inline int backup_bitmap_words(const Arena &A) { return A.pc ? (A.M + 31) / 32 : 0; }
static inline size_t backup_smem(const Arena &A) { return (size_t)4 * backup_bitmap_words(A) * sizeof(unsigned); }

// temporary device buffers of the standalone entry points: freed on every return path
struct Scratch {
    std::vector<void *> bufs;
    ~Scratch() { for (void *q : bufs) cudaFree(q); }
    template <typename T> cudaError_t get(T **out, size_t bytes) {
        void *q = nullptr;
        cudaError_t err = cudaMalloc(&q, bytes ? bytes : 1);
        if (err == cudaSuccess) { bufs.push_back(q); *out = (T *)q; }
        return err;
    }
};

static void dfree(b200_engine *e, void *p) {   // release one engine-owned allocation early (a buffer that is being replaced)
    if (!p) return;
    for (size_t i = 0; i < e->allocs.size(); ++i)
        if (e->allocs[i] == p) { e->allocs.erase(e->allocs.begin() + i); break; }
    cudaFree(p);
}

template <typename T>
static int dalloc(b200_engine *e, T **p, size_t n, bool zero = true) {
    void *q = nullptr;
    cudaError_t err = cudaMalloc(&q, n * sizeof(T));
    if (err != cudaSuccess) return fail(B200_ERR_CUDA, std::string("cudaMalloc ") + std::to_string(n * sizeof(T)) + " B: " + cudaGetErrorString(err));
    if (zero) cudaMemsetAsync(q, 0, n * sizeof(T), e->stream);
    e->allocs.push_back(q);
    *p = (T *)q;
    return 0;
}

// SPEC §2-4 fresh games, produced ON THE DEVICE so that no host restatement of the env exists in this library.
// seeds == nullptr: every game gets the default seed (SPEC §4); reset != 0: SPEC §4 reset() of the records in place.
__global__ void k_new_games(uint32_t *recs, int n, int app, int scoring, int randomizer, const uint32_t *seeds, int reset) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Game g;
    uint32_t w[REC_WORDS];
    if (reset) {
        load_rec(recs + (size_t)i * REC_WORDS, w);
        unpack(g, w);
        reset_game(g);
    } else {
        for (int q = 0; q < 10; ++q) g.w[q] = 0;
        g.piece = 0; g.rot = 0; g.px = 3; g.py = 0; g.bag = 0x7fu; g.dropcnt = 0; g.end = 0;
        g.app = app < 1 ? 1 : (app > 255 ? 255 : app); g.scoring = scoring ? 1 : 0; g.randomizer = randomizer ? 1 : 0;
        uint32_t seed = seeds ? seeds[i] : 0u;
        g.combo = 0; g.rng = seed ? seed : 0x9E3779B9u; g.score = 0; g.lines = 0;
        for (int q = 0; q < 4; ++q) g.ls[q] = 0;
        spawn(g);
    }
    pack(g, w);
    store_rec(recs + (size_t)i * REC_WORDS, w);
}

struct PhaseTimer {
    b200_engine *e; int ph;
    PhaseTimer(b200_engine *e_, int ph_) : e(e_), ph(ph_) {
        e->phase_launches[ph] += 1;
        if (!e->timing) return;
        if (e->ev_used + 2 > e->ev.size()) {
            size_t old = e->ev.size();
            e->ev.resize(old + 4096);
            for (size_t i = old; i < e->ev.size(); ++i) cudaEventCreate(&e->ev[i]);
        }
        cudaEventRecord(e->ev[e->ev_used], e->stream);
    }
    ~PhaseTimer() {
        if (!e->timing) return;
        cudaEventRecord(e->ev[e->ev_used + 1], e->stream);
        e->ev_phase.push_back(ph);
        e->ev_used += 2;
    }
};

static void flush_timing(b200_engine *e) {
    if (!e->timing || e->ev_used == 0) return;
    cudaStreamSynchronize(e->stream);
    for (size_t i = 0; i < e->ev_used; i += 2) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e->ev[i], e->ev[i + 1]);
        e->phase_ms[e->ev_phase[i / 2]] += ms;
    }
    e->ev_used = 0; e->ev_phase.clear();
}

extern "C" int b200_engine_create(const b200_config *cfg, b200_engine **out) {
    if (!cfg || !out) return fail(B200_ERR_BAD_ARG, "null argument");
    if (cfg->n_games < 1 || cfg->max_nodes < 16 || cfg->max_nodes >= (1 << 28) || (cfg->max_nodes & 3))
        return fail(B200_ERR_BAD_ARG, "n_games >= 1, 16 <= max_nodes < 2^28, max_nodes % 4 == 0");
    if (cfg->mode < 0 || cfg->mode > 3) return fail(B200_ERR_BAD_ARG, "mode");
    if (cfg->mode == MODE_DIST && (cfg->dist_bins < 2 || cfg->dist_bins > 64 || !(cfg->dist_vmax > cfg->dist_vmin)))
        return fail(B200_ERR_BAD_ARG, "distributional mode needs 2 <= dist_bins <= 64 and dist_vmax > dist_vmin");
    if (cfg->mode == MODE_DIST && cfg->eval_kind == B200_EVAL_NET_FP16)
        return fail(B200_ERR_BAD_ARG, "eval_kind net_fp16 has no distributional network: use net_tc or net in B200_MODE_DIST");
    if (cfg->mode == MODE_VANILLA && cfg->eval_kind == B200_EVAL_EXTERNAL)
        return fail(B200_ERR_BAD_ARG, "eval_kind external needs B200_MODE_LP, B200_MODE_SINGLE or B200_MODE_DIST (Vanilla evaluates by rollout)");
    if (cfg->mode != MODE_VANILLA && cfg->eval_kind == B200_EVAL_EXTERNAL_GAME)
        return fail(B200_ERR_BAD_ARG, "eval_kind external_game evaluates leaf games and needs B200_MODE_VANILLA: use eval_kind external "
                                      "for a board evaluator in B200_MODE_LP, B200_MODE_SINGLE or B200_MODE_DIST");
    if (cfg->mode != MODE_DIST && cfg->eval_kind == B200_EVAL_DIST_FP16)
        return fail(B200_ERR_BAD_ARG, "eval_kind dist_fp16 is the distributional network's one-term form and needs B200_MODE_DIST: "
                                      "use net_fp16 for the value network");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    CK(cudaSetDevice(cfg->device));
    b200_engine *e = new b200_engine();
    struct Guard { b200_engine *e; ~Guard() { if (e) b200_engine_destroy(e); } } guard{e};   // every failing return below destroys the half-built engine
    e->cfg = *cfg;
    CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, cfg->device));
    e->n_sm = prop.multiProcessorCount;
    Arena &A = e->A;
    memset(&A, 0, sizeof(A));
    A.G = cfg->n_games; A.M = cfg->max_nodes;
    int H = A.M + A.M / 2;                       // load factor <= 2/3 (tombstones only live inside k_gc, which rebuilds both tables)
    if (H < 16) H = 16;
    A.H = H; A.trace_max = cfg->trace_max > 0 ? cfg->trace_max : 512;
    A.mode = cfg->mode; A.low = cfg->low; A.lp_end_from_obs = cfg->lp_end_from_obs; A.lp_var_gamma2 = cfg->lp_var_gamma2;
    A.stale_pop = cfg->stale_pop; A.eval_kind = cfg->eval_kind; A.overflow_reset = cfg->overflow_reset; A.gc_min_gain = cfg->overflow_reset ? cfg->max_nodes / 8 : 0; A.gamma = cfg->gamma; A.rollout_variance = cfg->rollout_variance;
    size_t GM = (size_t)A.G * A.M, G = (size_t)A.G;
    int rc = 0;
    rc |= dalloc(e, &A.row, GM * ROW_WORDS);
    rc |= dalloc(e, &A.stat, GM);
    rc |= dalloc(e, &A.rec, GM * REC_WORDS, false);
    rc |= dalloc(e, &A.key, GM * KEY_WORDS);
    rc |= dalloc(e, &A.ntab, G * H);
    rc |= dalloc(e, &A.otab, G * H);
    rc |= dalloc(e, &A.nfree, GM); rc |= dalloc(e, &A.ofree, GM);
    rc |= dalloc(e, &A.n_nfree, G); rc |= dalloc(e, &A.n_ofree, G);
    rc |= dalloc(e, &A.root, G); rc |= dalloc(e, &A.episode, G); rc |= dalloc(e, &A.status, G); rc |= dalloc(e, &A.srng, G);
    rc |= dalloc(e, &A.trace, G * A.trace_max); rc |= dalloc(e, &A.trace_len, G); rc |= dalloc(e, &A.leaf_kind, G);
    rc |= dalloc(e, &A.trace_meta, G * A.trace_max);
    {   // collection scratch: one set per k_gc CTA (gc_blocks), not per game
        e->gc_pool_main = e->n_sm * 4 < A.G ? e->n_sm * 4 : A.G;
        const size_t pool = (size_t)(e->gc_pool_main + DEEP_GC_BLOCKS) * A.M;
        rc |= dalloc(e, &A.nmark, pool); rc |= dalloc(e, &A.omark, pool); rc |= dalloc(e, &A.gc_queue, pool * 2);
    }
    rc |= dalloc(e, &A.cur, G * REC_WORDS);
    rc |= dalloc(e, &A.req, G * 8); rc |= dalloc(e, &A.n_req, 4);
    rc |= dalloc(e, &A.gc_list, G); rc |= dalloc(e, &A.pending, G); rc |= dalloc(e, &A.resume_a, G);
    rc |= dalloc(e, &A.eval_out, G * 8); rc |= dalloc(e, &A.rollout_val, G);
    rc |= dalloc(e, &A.counters, 48);
    A.fin_cap = 4 * A.G;
    rc |= dalloc(e, &A.fin_log, (size_t)A.fin_cap * 4); rc |= dalloc(e, &A.fin_count, 1);
    if (cfg->mode == MODE_DIST) {
        A.dist_bins = cfg->dist_bins; A.dist_vmin = cfg->dist_vmin; A.dist_vmax = cfg->dist_vmax;
        rc |= dalloc(e, &A.nstat, GM * NSTAT_WORDS); rc |= dalloc(e, &A.ndist, GM * (size_t)A.dist_bins); rc |= dalloc(e, &A.dist_eval, G * (size_t)A.dist_bins);
    }
    if (cfg->eval_kind == B200_EVAL_EXTERNAL) {
        rc |= dalloc(e, &e->d_ext_mark, G * 8); rc |= dalloc(e, &e->d_ext_rows, G * 8); rc |= dalloc(e, &e->d_ext_n, 1);
    }
    if (cfg->eval_kind == B200_EVAL_EXTERNAL_GAME) {
        rc |= dalloc(e, &e->d_ext_rows, G); rc |= dalloc(e, &e->d_ext_n, 1); rc |= dalloc(e, &A.rollout_var, G);
    }
    rc |= dalloc(e, &e->d_default_rec, REC_WORDS);
    rc |= dalloc(e, &e->d_stats, G * 21); rc |= dalloc(e, &e->d_action, G);
    e->d_game_stats = A.counters + 8;
    float *zt = nullptr;
    rc |= dalloc(e, &zt, ZTABLE_N);
    if (rc) return B200_ERR_CUDA;
    {   // z(n) = norm_quantile(n) narrowed to float: special.h:26-33 + core.h:93, evaluated with the host libm
        std::vector<float> h(ZTABLE_N);
        const double l2 = log(2.0), l22 = log(22.0), l41 = log(41.0);
        for (int n = 0; n < ZTABLE_N; ++n) {
            double t = (double)n, alpha = 1 - 1 / t;
            h[n] = (float)(10 * log(1 - log(-log(alpha) / l2) / l22) / l41);
        }
        CK(cudaMemcpyAsync(zt, h.data(), ZTABLE_N * sizeof(float), cudaMemcpyHostToDevice, e->stream));
        CK(cudaStreamSynchronize(e->stream));
        A.ztable = zt;
    }
    k_new_games<<<1, 1, 0, e->stream>>>(e->d_default_rec, 1, cfg->actions_per_drop, cfg->scoring, cfg->randomizer, nullptr, 0);
    k_init_arena<<<e->n_sm * 8, 256, 0, e->stream>>>(A, e->d_default_rec, cfg->seed);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    guard.e = nullptr;
    *out = e;
    return B200_OK;
}

extern "C" int b200_engine_destroy(b200_engine *e) {
    if (!e) return B200_OK;
    cudaSetDevice(e->cfg.device);                    // the current device is per host thread: this one may not have made it current
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->step_exec) cudaGraphExecDestroy(e->step_exec);
    tc_destroy(e->tc_state);
    dn_tc_destroy(e->dn_tc_state);
    for (void *p : e->allocs) cudaFree(p);
    for (auto &ev : e->ev) cudaEventDestroy(ev);
    if (e->t0) { cudaEventDestroy(e->t0); cudaEventDestroy(e->t1); }
    if (e->stream1) cudaStreamDestroy(e->stream1);
    if (e->ev_fork) { cudaEventDestroy(e->ev_fork); cudaEventDestroy(e->ev_join); }
    if (e->stream && e->own_stream) cudaStreamDestroy(e->stream);
    delete e;
    return B200_OK;
}

// SURVEY 8(b).5 "explicit cudaStream_t": all work of the engine is issued on `cuda_stream` from now on (nullptr: a private non-blocking
// stream again).  The engine drains its current stream first, so nothing of it is in flight on two streams at once; the captured
// simulation step is dropped and re-captured on the new stream.  The caller keeps ownership of its stream and must keep it alive.
extern "C" int b200_engine_set_stream(b200_engine *e, void *cuda_stream) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    REFUSE_IF_OPEN(e, "b200_engine_set_stream");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaStreamSynchronize(e->stream));
    if (e->stream1) CK(cudaStreamSynchronize(e->stream1));
    drop_step_graph(e);
    cudaStream_t ns = (cudaStream_t)cuda_stream;
    const bool own = ns == nullptr;
    if (own) CK(cudaStreamCreateWithFlags(&ns, cudaStreamNonBlocking));
    if (e->own_stream) cudaStreamDestroy(e->stream);
    e->stream = ns; e->own_stream = own;
    return B200_OK;
}

extern "C" int b200_engine_get_stream(b200_engine *e, void **cuda_stream_out) {
    if (!e || !cuda_stream_out) return fail(B200_ERR_BAD_ARG, "null argument");
    *cuda_stream_out = (void *)e->stream;
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- weights
// net_tc and net_fp16 run the same tensor-core kernels and weight layout, with two fp16 terms per operand or one (valuenet_tc.cuh)
static bool tc_net(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_NET_TC || e->cfg.eval_kind == B200_EVAL_NET_FP16; }
static decltype(&k_tc_conv<2>) tc_conv_kernel(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_NET_FP16 ? k_tc_conv<1> : k_tc_conv<2>; }
static decltype(&k_tc_fc<2>) tc_fc_kernel(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_NET_FP16 ? k_tc_fc<1> : k_tc_fc<2>; }
static decltype(&k_tc_fc_dbg<2>) tc_fc_dbg_kernel(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_NET_FP16 ? k_tc_fc_dbg<1> : k_tc_fc_dbg<2>; }

extern "C" int b200_load_weights(b200_engine *e, const float *w) {
    if (!e || !w) return fail(B200_ERR_BAD_ARG, "null argument");
    REFUSE_IF_EXT(e, "b200_load_weights");
    if (e->cfg.eval_kind == B200_EVAL_DIST_FP16) return fail(B200_ERR_BAD_ARG, "eval_kind dist_fp16 has no value network (use net_fp16)");
    if (tc_net(e) && !tc_weights_fit(w))
        return fail(B200_ERR_BAD_ARG, e->cfg.eval_kind == B200_EVAL_NET_TC
                    ? "net_tc: a conv or fc1 weight is non-finite or has |w| * 64 > 65504, which overflows the tensor cores' "
                      "fp16 x 2 operand split (eval_kind net takes finite weights of any size)"
                    : "net_fp16: a conv or fc1 weight is non-finite or has |w| * 64 > 65504, which overflows the tensor cores' "
                      "scaled fp16 operands (eval_kind net takes finite weights of any size)");
    CK(cudaSetDevice(e->cfg.device));
    const float *c1w = w, *c1b = c1w + 288, *c2w = c1b + 32, *c2b = c2w + 9216, *c3w = c2b + 32, *c3b = c3w + 9216;
    const float *f1w = c3b + 32, *f1b = f1w + 458752, *fow = f1b + 256, *fob = fow + 512, *ub = fob + 2, *lb = ub + 2;
    // pure re-layout (no arithmetic): see NetWeights
    std::vector<float> h;
    h.resize(288 + 9216 * 2 + 96 + (size_t)1792 * 256 + 256 + 512 + 6);
    float *p = h.data();
    float *w1 = p; p += 288;
    float *w2 = p; p += 9216;
    float *w3 = p; p += 9216;
    float *b123 = p; p += 96;
    float *wf = p; p += (size_t)1792 * 256;
    float *bf = p; p += 256;
    float *wo = p; p += 512;
    float *tail = p;
    for (int co = 0; co < 32; ++co)
        for (int tap = 0; tap < 9; ++tap) w1[tap * 32 + co] = c1w[co * 9 + tap];
    for (int co = 0; co < 32; ++co)
        for (int ci = 0; ci < 32; ++ci)
            for (int tap = 0; tap < 9; ++tap) {
                w2[(ci * 9 + tap) * 32 + co] = c2w[(co * 32 + ci) * 9 + tap];
                w3[(ci * 9 + tap) * 32 + co] = c3w[(co * 32 + ci) * 9 + tap];
            }
    memcpy(b123, c1b, 128); memcpy(b123 + 32, c2b, 128); memcpy(b123 + 64, c3b, 128);
    for (int n = 0; n < 256; ++n)
        for (int c = 0; c < 32; ++c)
            for (int y = 0; y < 14; ++y)
                for (int x = 0; x < 4; ++x) wf[(size_t)((y * 32 + c) * 4 + x) * 256 + n] = f1w[(size_t)n * 1792 + c * 56 + y * 4 + x];
    memcpy(bf, f1b, 1024); memcpy(wo, fow, 2048);
    tail[0] = fob[0]; tail[1] = fob[1]; tail[2] = ub[0]; tail[3] = ub[1]; tail[4] = lb[0]; tail[5] = lb[1];
    if (!e->d_wraw) { if (dalloc(e, &e->d_wraw, h.size(), false)) return B200_ERR_CUDA; }
    CK(cudaMemcpyAsync(e->d_wraw, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    float *d = e->d_wraw;
    e->W.w1 = d; e->W.w2 = d + 288; e->W.w3 = d + 288 + 9216; e->W.b1 = d + 288 + 18432; e->W.b2 = e->W.b1 + 32; e->W.b3 = e->W.b1 + 64;
    e->W.wfc1 = e->W.b1 + 96; e->W.bfc1 = e->W.wfc1 + (size_t)1792 * 256; e->W.wout = e->W.bfc1 + 256;
    e->W.bout = e->W.wout + 512; e->W.ub = e->W.bout + 2; e->W.lb = e->W.bout + 4;
    CK(cudaFuncSetAttribute(k_vn_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, VN_SMEM_BYTES));
    CK(cudaFuncSetAttribute(k_vn_conv_dbg, cudaFuncAttributeMaxDynamicSharedMemorySize, VN_SMEM_BYTES));
    {
        int rc = tc_prepare(&e->tc_state, w, e->stream);
        if (rc) return fail(B200_ERR_CUDA, "tensor-core weight preparation failed");
    }
    e->have_weights = true;
    e->h_w.assign(w, w + B200_N_WEIGHTS);
    drop_step_graph(e);
    return B200_OK;
}

static int ensure_act3(b200_engine *e, size_t rows) {
    if (e->act3_rows >= rows) return 0;
    if (e->d_act3) { cudaStreamSynchronize(e->stream); dfree(e, e->d_act3); e->d_act3 = nullptr; e->act3_rows = 0; }
    if (dalloc(e, &e->d_act3, rows * 1792, false)) return B200_ERR_CUDA;
    e->act3_rows = rows;
    return 0;
}

// run the network over the request list req[0..*n_req) -> eval_out; device-side count, no host sync.  dbg (standalone requests only):
// run the DBG instantiations instead, which also copy act1 / act2 there (tensor-core kinds: k_tc_conv_dbg, TCC_DBG_BYTES per request;
// net: k_vn_conv_dbg, VN_DBG_FLOATS floats per request) and fc1's fp32 accumulator to dbg_fc (256 floats per request)
static int launch_net(b200_engine *e, const uint2 *req, const int32_t *n_req, const uint32_t *keys, int M, float2 *eval_out,
                      size_t max_rows, uint8_t *dbg = nullptr, float *dbg_fc = nullptr) {
    if (!e->have_weights) return fail(B200_ERR_NO_WEIGHTS, "b200_load_weights was not called");
    if (tc_net(e)) {
        TcState *st = (TcState *)e->tc_state;
        const uint8_t *act3_before = st->d_act3;
        if (tc_ensure_act3(st, max_rows, e->stream)) return fail(B200_ERR_CUDA, "act3 (tensor-core layout) allocation failed");
        if (act3_before && st->d_act3 != act3_before) drop_step_graph(e);   // a larger standalone batch moved the activation buffer
        if (dbg) {
            (e->cfg.eval_kind == B200_EVAL_NET_FP16 ? k_tc_conv_dbg<1> : k_tc_conv_dbg<2>)<<<e->n_sm, TCC_THREADS, TCC_SMEM, e->stream>>>(
                e->W, st->TW, req, n_req, keys, st->d_act3, (int)st->tiles, dbg);
        } else {
            PhaseTimer t(e, PH_CONV);
            tc_conv_kernel(e)<<<e->n_sm, TCC_THREADS, TCC_SMEM, e->stream>>>(e->W, st->TW, req, n_req, nullptr, keys, M, st->d_act3, (int)st->tiles,
                                                                             e->timing ? e->A.counters + 16 : nullptr);
        }
        if (dbg) {
            tc_fc_dbg_kernel(e)<<<e->n_sm, TCF_THREADS, TCF_SMEM, e->stream>>>(e->W, st->TW, st->d_act3, (int)st->tiles, req, n_req, eval_out, dbg_fc);
        } else {
            PhaseTimer t(e, PH_FC);
            tc_fc_kernel(e)<<<e->n_sm, TCF_THREADS, TCF_SMEM, e->stream>>>(e->W, st->TW, st->d_act3, (int)st->tiles, req, n_req, eval_out);
        }
        CK(cudaGetLastError());
        return B200_OK;
    }
    {
        const float *act3_before = e->d_act3;
        if (ensure_act3(e, max_rows)) return B200_ERR_CUDA;
        if (act3_before && e->d_act3 != act3_before) drop_step_graph(e);
    }
    if (dbg) {
        k_vn_conv_dbg<<<e->n_sm, VN_THREADS, VN_SMEM_BYTES, e->stream>>>(e->W, req, n_req, keys, M, e->d_act3, reinterpret_cast<float *>(dbg));
        k_vn_fc_dbg<<<e->n_sm * 2, FC_THREADS, 0, e->stream>>>(e->W, e->d_act3, req, n_req, eval_out, dbg_fc);
        CK(cudaGetLastError());
        return B200_OK;
    }
    {
        PhaseTimer t(e, PH_CONV);
        k_vn_conv<<<e->n_sm, VN_THREADS, VN_SMEM_BYTES, e->stream>>>(e->W, req, n_req, keys, M, e->d_act3);
    }
    {
        PhaseTimer t(e, PH_FC);
        k_vn_fc<<<e->n_sm * 2, FC_THREADS, 0, e->stream>>>(e->W, e->d_act3, req, n_req, eval_out);
    }
    CK(cudaGetLastError());
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- distributional network
__global__ void k_states_to_keys(const int8_t *states, int k, uint32_t *keys, uint2 *req);   // defined with the standalone value net below

// net_tc and dist_fp16 run the same tensor-core distributional kernels and weight layout, with two fp16 terms per operand or one (distnet_tc.cuh)
static bool dn_tc_net(const b200_engine *e) { return e->cfg.eval_kind == B200_EVAL_NET_TC || e->cfg.eval_kind == B200_EVAL_DIST_FP16; }
// floats of model_distributional.py's state_dict vector: conv1, conv2, fc1, fc_v (weights and biases)
static size_t dn_weight_count(int atoms) { return (size_t)512 + 32 + 16384 + 32 + 128 * 2048 + 128 + (size_t)atoms * 128 + atoms; }

extern "C" int b200_load_dist_weights(b200_engine *e, const float *w, int atoms) {
    if (!e || !w || atoms < 2 || atoms > 64) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_EXT(e, "b200_load_dist_weights");
    if (e->cfg.eval_kind == B200_EVAL_NET_FP16) return fail(B200_ERR_BAD_ARG, "eval_kind net_fp16 has no distributional network");
    CK(cudaSetDevice(e->cfg.device));
    if (e->A.mode == MODE_DIST && atoms != e->A.dist_bins) return fail(B200_ERR_BAD_ARG, "atoms must equal dist_bins");
    if (e->cfg.eval_kind == B200_EVAL_NET_TC && !dn_tc_weights_fit(w))
        return fail(B200_ERR_BAD_ARG, "net_tc: a conv or fc1 weight is non-finite or has |w| * 64 > 65504, which overflows the tensor cores' "
                                      "fp16 x 2 operand split (eval_kind net takes finite weights of any size)");
    if (e->cfg.eval_kind == B200_EVAL_DIST_FP16 && !dn_tc_weights_fit(w))
        return fail(B200_ERR_BAD_ARG, "dist_fp16: a conv or fc1 weight is non-finite or has |w| * 64 > 65504, which overflows the tensor cores' "
                                      "scaled fp16 operands (eval_kind net takes finite weights of any size)");
    std::vector<float> h;
    dn_relayout(w, atoms, h);
    if (!e->d_dnw) { if (dalloc(e, &e->d_dnw, h.size(), false)) return B200_ERR_CUDA; }
    CK(cudaMemcpyAsync(e->d_dnw, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->DW = dn_pointers(e->d_dnw, atoms);
    CK(cudaFuncSetAttribute(k_dn_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, DN_CONV_SMEM));
    CK(cudaFuncSetAttribute(k_dn_fc, cudaFuncAttributeMaxDynamicSharedMemorySize, DN_FC_SMEM));
    CK(cudaFuncSetAttribute(k_dn_conv_dbg, cudaFuncAttributeMaxDynamicSharedMemorySize, DN_CONV_SMEM));
    CK(cudaFuncSetAttribute(k_dn_fc_dbg, cudaFuncAttributeMaxDynamicSharedMemorySize, DN_FC_SMEM));
    if (dn_tc_prepare(&e->dn_tc_state, w, atoms, e->stream)) return fail(B200_ERR_CUDA, "tensor-core weight preparation (distributional network) failed");
    e->have_dist_weights = true;
    e->h_dnw.assign(w, w + dn_weight_count(atoms)); e->dn_atoms = atoms;   // the state_dict vector dn_relayout reads
    drop_step_graph(e);
    return B200_OK;
}

// dbg (standalone requests only): run the DBG instantiations instead, which also copy act1 there (tensor-core kinds: k_tdc_conv_dbg,
// TDC_ASLOT per request; net: k_dn_conv_dbg, DN_DBG_A1 floats per request) and fc1's fp32 accumulator to dbg_fc (128 floats per
// request); net's k_dn_fc_dbg also copies the logits to dbg_lg (atoms floats per request)
static int launch_distnet_on(b200_engine *e, const uint2 *req, const int32_t *n_req, const uint32_t *keys, int M, float *out, size_t max_rows,
                             uint8_t *dbg = nullptr, float *dbg_fc = nullptr, float *dbg_lg = nullptr) {
    if (!e->have_dist_weights) return fail(B200_ERR_NO_WEIGHTS, "b200_load_dist_weights was not called");
    if (dn_tc_net(e)) {
        DnTcState *st = (DnTcState *)e->dn_tc_state;
        bool moved = false;
        if (dn_tc_ensure_act2(st, max_rows, e->stream, &moved)) return fail(B200_ERR_CUDA, "act2 (tensor-core layout) allocation failed");
        if (moved) drop_step_graph(e);
        const bool one = e->cfg.eval_kind == B200_EVAL_DIST_FP16;
        if (dbg) {
            (one ? k_tdc_conv_dbg<1> : k_tdc_conv_dbg<2>)<<<e->n_sm, TDC_THREADS, TDC_SMEM, e->stream>>>(e->DW, st->TW, req, n_req, keys, st->d_act2,
                                                                                                       (int)st->tiles, dbg);
        } else {
            PhaseTimer t(e, PH_CONV);
            (one ? k_tdc_conv<1> : k_tdc_conv<2>)<<<e->n_sm, TDC_THREADS, TDC_SMEM, e->stream>>>(e->DW, st->TW, req, n_req, keys, M, st->d_act2,
                                                                                               (int)st->tiles);
        }
        if (dbg) {
            (one ? k_tdc_fc_dbg<1> : k_tdc_fc_dbg<2>)<<<e->n_sm, TDF_THREADS, TDF_SMEM, e->stream>>>(e->DW, st->TW, st->d_act2, (int)st->tiles, req, n_req,
                                                                                                   out, dbg_fc);
        } else {
            PhaseTimer t(e, PH_FC);
            (one ? k_tdc_fc<1> : k_tdc_fc<2>)<<<e->n_sm, TDF_THREADS, TDF_SMEM, e->stream>>>(e->DW, st->TW, st->d_act2, (int)st->tiles, req, n_req, out);
        }
        CK(cudaGetLastError());
        return B200_OK;
    }
    if (e->dn_rows < max_rows) {
        const bool had = e->d_dn_act != nullptr;
        if (had) { cudaStreamSynchronize(e->stream); dfree(e, e->d_dn_act); e->d_dn_act = nullptr; e->dn_rows = 0; }
        if (dalloc(e, &e->d_dn_act, max_rows * 2048, false)) return B200_ERR_CUDA;
        e->dn_rows = max_rows;
        if (had) drop_step_graph(e);
    }
    if (dbg) {
        k_dn_conv_dbg<<<e->n_sm * 2, DN_THREADS, DN_CONV_SMEM, e->stream>>>(e->DW, req, n_req, keys, M, e->d_dn_act, reinterpret_cast<float *>(dbg));
        k_dn_fc_dbg<<<e->n_sm, DN_THREADS, DN_FC_SMEM, e->stream>>>(e->DW, e->d_dn_act, req, n_req, out, dbg_fc, dbg_lg);
        CK(cudaGetLastError());
        return B200_OK;
    }
    {
        PhaseTimer t(e, PH_CONV);
        k_dn_conv<<<e->n_sm * 2, DN_THREADS, DN_CONV_SMEM, e->stream>>>(e->DW, req, n_req, keys, M, e->d_dn_act);
    }
    {
        PhaseTimer t(e, PH_FC);
        k_dn_fc<<<e->n_sm, DN_THREADS, DN_FC_SMEM, e->stream>>>(e->DW, e->d_dn_act, req, n_req, out);
    }
    CK(cudaGetLastError());
    return B200_OK;
}
static int launch_distnet(b200_engine *e) {
    return launch_distnet_on(e, e->A.req, e->A.n_req, e->A.key, e->A.M, e->A.dist_eval, (size_t)e->A.G);
}

// Model.inference of model/model_distributional.py (softmax over atoms): states[k][200] int8 -> dist[k][atoms]
static int distnet_forward(b200_engine *e, const int8_t *states, int k, int atoms, float *dist, uint8_t *dbg, float *dbg_fc,
                           float *dbg_lg = nullptr) {
    if (!e || !states || !dist || k < 1 || atoms != e->DW.atoms) return fail(B200_ERR_BAD_ARG, "bad argument (atoms must match the loaded weights)");
    CK(cudaSetDevice(e->cfg.device));
    int8_t *d_states = nullptr; uint32_t *d_keys = nullptr; uint2 *d_req = nullptr; int32_t *d_n = nullptr; float *d_out = nullptr;
    Scratch tmp;
    CK(tmp.get(&d_states, (size_t)k * 200)); CK(tmp.get(&d_keys, (size_t)k * KEY_WORDS * 4)); CK(tmp.get(&d_req, (size_t)k * 8));
    CK(tmp.get(&d_n, 4)); CK(tmp.get(&d_out, (size_t)k * atoms * 4));
    CK(cudaMemcpyAsync(d_states, states, (size_t)k * 200, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d_n, &k, 4, cudaMemcpyHostToDevice, e->stream));
    k_states_to_keys<<<(k + 127) / 128, 128, 0, e->stream>>>(d_states, k, d_keys, d_req);
    k_dn_req_rows<<<(k + 127) / 128, 128, 0, e->stream>>>(d_req, k);      // request i -> output row i
    int rc = launch_distnet_on(e, d_req, d_n, d_keys, 0, d_out, (size_t)k, dbg, dbg_fc, dbg_lg);
    if (rc == B200_OK) {
        cudaError_t ce = cudaMemcpyAsync(dist, d_out, (size_t)k * atoms * 4, cudaMemcpyDeviceToHost, e->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
        if (ce != cudaSuccess) rc = fail(B200_ERR_CUDA, cudaGetErrorString(ce));
    }
    cudaStreamSynchronize(e->stream);
    return rc;
}
extern "C" int b200_distnet_forward(b200_engine *e, const int8_t *states, int k, int atoms, float *dist) {
    if (e) REFUSE_IF_EXT(e, "b200_distnet_forward");
    return distnet_forward(e, states, k, atoms, dist, nullptr, nullptr);
}

// ---------------------------------------------------------------------------------------------------- games / roots
static inline int blocks_groups(int G) { return (G + GROUPS_PER_BLOCK - 1) / GROUPS_PER_BLOCK; }
static inline int gc_blocks(b200_engine *e) { int b = e->n_sm * 4; return e->A.G < b ? e->A.G : b; }

static int check_status(b200_engine *e) {   // cheap: max over the status array computed on the host after a small copy
    std::vector<int32_t> st(e->A.G);
    CK(cudaMemcpyAsync(st.data(), e->A.status, st.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    for (int g = 0; g < e->A.G; ++g)
        if (st[g] != ST_OK && !((st[g] == ST_ARENA_FULL || st[g] == ST_RESET_DONE) && e->A.overflow_reset)) {
            int code = st[g] == ST_ARENA_FULL ? B200_ERR_ARENA_FULL : B200_ERR_TRACE_FULL;
            return fail(code, "game " + std::to_string(g) + (st[g] == ST_ARENA_FULL ? ": arena full after garbage collection (raise max_nodes)" : ": trace longer than trace_max"));
        }
    return B200_OK;
}

// TreeAgent.remove_nodes() (agents/agent.py:246-257) for every game with fewer than min_free free node slots, as ONE batched k_gc
extern "C" int b200_remove_nodes(b200_engine *e, int min_free) {
    if (!e || min_free < 0) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_OPEN(e, "b200_remove_nodes");
    CK(cudaSetDevice(e->cfg.device));
    {
        PhaseTimer t(e, PH_GC);
        CK(cudaMemsetAsync(e->A.n_req + 1, 0, sizeof(int32_t), e->stream));
        k_gc_request<<<(e->A.G + 127) / 128, 128, 0, e->stream>>>(e->A, min_free);
        k_gc<<<gc_blocks(e), GC_THREADS, 0, e->stream>>>(e->A);
    }
    CK(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_set_gc_headroom(b200_engine *e, int min_free) {
    if (!e || min_free < 0) return fail(B200_ERR_BAD_ARG, "bad argument");
    e->gc_headroom = min_free;
    return B200_OK;
}

// Path cache (search_dev.cuh "path cache"): scheduling/memory-traffic only, no effect on any result.  LP mode, max_nodes <= 65536.
extern "C" int b200_set_path_cache(b200_engine *e, int on) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    REFUSE_IF_OPEN(e, "b200_set_path_cache");
    CK(cudaSetDevice(e->cfg.device));
    if (on) {
        if (e->A.mode != MODE_LP) return fail(B200_ERR_BAD_ARG, "the path cache serves B200_MODE_LP (its coherence rules rest on the LP backup)");
        if (e->A.M > PC_MAX_NODES) return fail(B200_ERR_BAD_ARG, "the path cache needs max_nodes <= 65536 (k_backup's bitmap of the trace's observations)");
    }
    CK(cudaStreamSynchronize(e->stream));
    drop_step_graph(e);
    if (on && !e->d_pc) {
        const size_t levels = (size_t)e->A.G * e->A.trace_max;
        if (dalloc(e, &e->d_pc, levels * 8, false) || dalloc(e, &e->d_pc_var, levels * 8, false) || dalloc(e, &e->d_pc_sib, levels, false) || dalloc(e, &e->d_pc_own, levels, false) ||
            dalloc(e, &e->d_pc_len, (size_t)e->A.G)) return B200_ERR_CUDA;
    }
    if (on) CK(cudaMemsetAsync(e->d_pc_len, 0, (size_t)e->A.G * sizeof(int32_t), e->stream));   // nothing is valid until a walk has left its entries
    e->A.pc = on ? e->d_pc : nullptr;
    e->A.pc_var = on ? e->d_pc_var : nullptr;
    e->A.pc_len = on ? e->d_pc_len : nullptr;
    e->A.pc_sib = on ? e->d_pc_sib : nullptr;
    e->A.pc_own = on ? e->d_pc_own : nullptr;
    return B200_OK;
}

extern "C" int b200_set_deep_lane(b200_engine *e, int max_games) {
    if (!e || max_games < 0 || max_games > e->A.G) return fail(B200_ERR_BAD_ARG, "0 <= max_games <= n_games");
    CK(cudaSetDevice(e->cfg.device));
    drop_step_graph(e);
    if (max_games > 0) {
        if (!e->stream1) {
            int lo = 0, hi = 0;
            CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            CK(cudaStreamCreateWithPriority(&e->stream1, cudaStreamNonBlocking, hi));      // the few deep CTAs go first wherever a slot frees up
            CK(cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming));
            if (dalloc(e, &e->d_glist0, (size_t)e->A.G) || dalloc(e, &e->d_nlist, 2) || dalloc(e, &e->d_nreq_deep, 2)) return B200_ERR_CUDA;
        }
        CK(cudaStreamSynchronize(e->stream));
        dfree(e, e->d_glist1); dfree(e, e->d_gc_list_deep); dfree(e, e->d_req_deep);
        e->d_glist1 = nullptr; e->d_gc_list_deep = nullptr; e->d_req_deep = nullptr;
        if (dalloc(e, &e->d_glist1, (size_t)max_games) || dalloc(e, &e->d_gc_list_deep, (size_t)max_games) || dalloc(e, &e->d_req_deep, (size_t)max_games * 8))
            return B200_ERR_CUDA;
        CK(cudaStreamSynchronize(e->stream));
    }
    e->deep_cap = max_games;
    return B200_OK;
}

static int update_root_impl(b200_engine *e, int auto_reset, bool headroom_collection) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    CK(cudaSetDevice(e->cfg.device));
    {
        PhaseTimer t(e, PH_MISC);
        CK(cudaMemsetAsync(e->A.n_req + 1, 0, sizeof(int32_t), e->stream));
        k_update_root<<<blocks_groups(e->A.G), TPB, 0, e->stream>>>(e->A, auto_reset, e->d_game_stats, 0);
        k_gc<<<gc_blocks(e), GC_THREADS, 0, e->stream>>>(e->A);                 // games whose free list ran dry (usually none)
        k_update_root<<<blocks_groups(e->A.G), TPB, 0, e->stream>>>(e->A, auto_reset, e->d_game_stats, 1);
    }
    if (headroom_collection && e->gc_headroom > 0) {
        int rc = b200_remove_nodes(e, e->gc_headroom);
        if (rc) return rc;
    }
    CK(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_update_root(b200_engine *e, int auto_reset) {
    if (e) REFUSE_IF_OPEN(e, "b200_update_root");
    return update_root_impl(e, auto_reset, true);
}

extern "C" int b200_set_games(b200_engine *e, const uint32_t *recs) {
    if (!e || !recs) return fail(B200_ERR_BAD_ARG, "null argument");
    REFUSE_IF_OPEN(e, "b200_set_games");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(e->A.cur, recs, (size_t)e->A.G * REC_WORDS * 4, cudaMemcpyHostToDevice, e->stream));
    int rc = update_root_impl(e, 0, false);   // handing the games over is not a move: the driver's between-moves collection (b200_set_gc_headroom) is not due here
    if (rc) return rc;
    return check_status(e);
}

extern "C" int b200_get_games(b200_engine *e, uint32_t *recs) {
    if (!e || !recs) return fail(B200_ERR_BAD_ARG, "null argument");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(recs, e->A.cur, (size_t)e->A.G * REC_WORDS * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- simulations
static bool deep_lane_on(const b200_engine *e) {
    return e->deep_cap > 0 && (e->A.mode == MODE_LP || e->A.mode == MODE_SINGLE) && tc_net(e);
}

// The step with the deep lane: the deepest games (k_classify, once per move) walk on stream1 while the others walk, collect AND run their
// network launch on the engine's stream; the lanes join, the deep lane's requests go behind the others' (k_merge_requests), a second, small
// k_tc_conv evaluates them, and k_tc_fc / k_backup work on all of them as before.  With phase timing on everything runs on one stream
// in the same order.  Which lane a game is in changes nothing in its results.
static int enqueue_step_lanes(b200_engine *e) {
    const Arena &A = e->A;
    const int G = A.G;
    if (!e->have_weights) return fail(B200_ERR_NO_WEIGHTS, "b200_load_weights was not called");
    TcState *st = (TcState *)e->tc_state;
    const uint8_t *act3_before = st->d_act3;
    if (tc_ensure_act3(st, (size_t)G * (A.mode == MODE_LP ? 7 : 1), e->stream)) return fail(B200_ERR_CUDA, "act3 (tensor-core layout) allocation failed");
    if (act3_before && st->d_act3 != act3_before) drop_step_graph(e);
    cudaStream_t s0 = e->stream, s1 = e->timing ? e->stream : e->stream1;
    Arena A0 = A, A1 = A;
    A0.glist = e->d_glist0; A0.n_list = e->d_nlist;
    A1.glist = e->d_glist1; A1.n_list = e->d_nlist + 1;
    A1.req = e->d_req_deep; A1.n_req = e->d_nreq_deep; A1.gc_list = e->d_gc_list_deep;
    A1.nmark += (size_t)e->gc_pool_main * A.M; A1.omark += (size_t)e->gc_pool_main * A.M; A1.gc_queue += (size_t)e->gc_pool_main * A.M * 2;
    A0.prof = e->timing ? A.counters + 32 : nullptr;
    CK(cudaMemsetAsync(A.n_req, 0, 4 * sizeof(int32_t), s0));
    CK(cudaMemsetAsync(e->d_nreq_deep, 0, 2 * sizeof(int32_t), s0));
    if (s1 != s0) { CK(cudaEventRecord(e->ev_fork, s0)); CK(cudaStreamWaitEvent(s1, e->ev_fork, 0)); }
    const int deep_groups = blocks_groups(e->deep_cap);
    {
        PhaseTimer t(e, PH_SELECT);
        k_select_expand<<<(G + GROUPS_PER_BLOCK - 1) / GROUPS_PER_BLOCK, TPB, 0, s0>>>(A0);
        k_select_expand<<<(e->deep_cap + GROUPS_PER_BLOCK - 1) / GROUPS_PER_BLOCK, TPB, 0, s1>>>(A1);
    }
    {
        PhaseTimer t(e, PH_GC);
        k_gc<<<gc_blocks(e), GC_THREADS, 0, s0>>>(A0);
        k_expand_resume<<<blocks_groups(G), TPB, 0, s0>>>(A0);
        k_gc<<<DEEP_GC_BLOCKS, GC_THREADS, 0, s1>>>(A1);
        k_expand_resume<<<deep_groups, TPB, 0, s1>>>(A1);
    }
    {
        PhaseTimer t(e, PH_CONV);
        tc_conv_kernel(e)<<<e->n_sm, TCC_THREADS, TCC_SMEM, s0>>>(e->W, st->TW, A.req, A.n_req, nullptr, A.key, A.M, st->d_act3, (int)st->tiles,
                                                                  e->timing ? A.counters + 16 : nullptr);
    }
    if (s1 != s0) { CK(cudaEventRecord(e->ev_join, s1)); CK(cudaStreamWaitEvent(s0, e->ev_join, 0)); }
    {
        PhaseTimer t(e, PH_CONV);
        k_merge_requests<<<1, 256, 0, s0>>>(A.req, A.n_req, e->d_req_deep, e->d_nreq_deep);
        tc_conv_kernel(e)<<<e->n_sm, TCC_THREADS, TCC_SMEM, s0>>>(e->W, st->TW, A.req, A.n_req, A.n_req + 2, A.key, A.M, st->d_act3, (int)st->tiles, nullptr);
    }
    {
        PhaseTimer t(e, PH_FC);
        tc_fc_kernel(e)<<<e->n_sm, TCF_THREADS, TCF_SMEM, s0>>>(e->W, st->TW, st->d_act3, (int)st->tiles, A.req, A.n_req, A.eval_out);
    }
    {
        PhaseTimer t(e, PH_BACKUP);
        k_backup<<<(G + 3) / 4, 128, backup_smem(A), s0>>>(A, backup_bitmap_words(A));
    }
    CK(cudaGetLastError());
    return B200_OK;
}

// The first half of a simulation step (one lane): select+expand, then the collections the step needs and the expansions they held up.
// Leaves the step's evaluation requests in A.req[0 .. *A.n_req).
static int step_select(b200_engine *e) {
    const Arena &A = e->A;
    const int G = A.G;
    CK(cudaMemsetAsync(A.n_req, 0, 2 * sizeof(int32_t), e->stream));
    {
        PhaseTimer t(e, PH_SELECT);
        Arena Ap = A;
        Ap.prof = e->timing ? A.counters + 32 : nullptr;
        k_select_expand<<<(G + GROUPS_PER_BLOCK - 1) / GROUPS_PER_BLOCK, TPB, 0, e->stream>>>(Ap);
    }
    {   // remove_nodes for the games that ran out of free slots in this step, then the rest of their expansion
        PhaseTimer t(e, PH_GC);
        k_gc<<<gc_blocks(e), GC_THREADS, 0, e->stream>>>(A);
        k_expand_resume<<<blocks_groups(G), TPB, 0, e->stream>>>(A);
    }
    return B200_OK;
}

// The second half: back every game's evaluated leaf up its trace (the evaluator's outputs are in A.eval_out / A.dist_eval / A.rollout_val).
static void step_backup(b200_engine *e) {
    const Arena &A = e->A;
    PhaseTimer t(e, PH_BACKUP);
    if (A.mode == MODE_DIST) k_dist_backup<<<(A.G + 3) / 4, 128, 0, e->stream>>>(A);
    else k_backup<<<(A.G + 3) / 4, 128, backup_smem(A), e->stream>>>(A, backup_bitmap_words(A));
}

// One simulation step of every game: select+expand -> (collect garbage, resume) -> evaluate -> backup.
static int enqueue_step(b200_engine *e) {
    const Arena &A = e->A;
    const int G = A.G;
    if (deep_lane_on(e)) return enqueue_step_lanes(e);
    int rc = step_select(e);
    if (rc) return rc;
    if (A.mode == MODE_VANILLA) {
        PhaseTimer t(e, PH_ROLLOUT);
        k_rollout<<<(G + 63) / 64, 64, 0, e->stream>>>(A);
    } else if (A.mode == MODE_DIST) {
        if (e->cfg.eval_kind == B200_EVAL_SYNTHETIC) {
            PhaseTimer t(e, PH_SYNTH);
            k_eval_synthetic_dist<<<(G + 127) / 128, 128, 0, e->stream>>>(A);
        } else {
            rc = launch_distnet(e);
            if (rc) return rc;
        }
    } else if (e->cfg.eval_kind == B200_EVAL_SYNTHETIC) {
        PhaseTimer t(e, PH_SYNTH);
        k_eval_synthetic<<<(G * 7 + 255) / 256 < 1184 ? (G * 7 + 255) / 256 : 1184, 256, 0, e->stream>>>(A);
    } else {
        rc = launch_net(e, A.req, A.n_req, A.key, A.M, A.eval_out, (size_t)G * (A.mode == MODE_LP ? 7 : 1));
        if (rc) return rc;
    }
    step_backup(e);
    return B200_OK;
}

// Capture one step (same launches, same arguments every step: all sizes are read on the device) and replay it.  The first
// step of an engine runs directly so that lazily allocated buffers (activations) exist before the capture.
static void capture_step(b200_engine *e) {
    uint64_t before[PH_N];
    for (int i = 0; i < PH_N; ++i) before[i] = e->phase_launches[i];
    cudaGraph_t graph = nullptr;
    if (cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); e->step_graph_failed = true; return; }
    int rc = enqueue_step(e);
    cudaError_t ce = cudaStreamEndCapture(e->stream, &graph);
    for (int i = 0; i < PH_N; ++i) { e->step_launches[i] = e->phase_launches[i] - before[i]; e->phase_launches[i] = before[i]; }
    if (rc == B200_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&e->step_exec, graph, 0) == cudaSuccess) {
        cudaGraphDestroy(graph);
        return;
    }
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    e->step_exec = nullptr; e->step_graph_failed = true;    // direct launches from now on
}

extern "C" int b200_run_sims(b200_engine *e, int sims) {
    if (!e || sims < 0) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_EXT(e, "b200_run_sims");
    CK(cudaSetDevice(e->cfg.device));
    const Arena &A = e->A;
    const bool need_net = A.mode != MODE_VANILLA && e->cfg.eval_kind != B200_EVAL_SYNTHETIC;
    if (need_net && !(A.mode == MODE_DIST ? e->have_dist_weights : e->have_weights)) return fail(B200_ERR_NO_WEIGHTS, "b200_load_weights was not called");
    CK(cudaMemsetAsync(A.counters + 12, 0, sizeof(unsigned long long), e->stream));   // counter 12: the longest trace of this call
    if (deep_lane_on(e) && sims > 0)     // this move's lanes, from the trace lengths of the previous move's last simulation
        k_classify<<<1, 1024, 0, e->stream>>>(A, e->deep_cap, e->d_glist0, e->d_nlist, e->d_glist1, e->d_nlist + 1);
    for (int s = 0; s < sims; ++s) {
        if (!e->timing && e->step_exec) {
            CK(cudaGraphLaunch(e->step_exec, e->stream));
            for (int i = 0; i < PH_N; ++i) e->phase_launches[i] += e->step_launches[i];
            continue;
        }
        int rc = enqueue_step(e);
        if (rc) return rc;
        if (!e->timing && !e->step_exec && !e->step_graph_failed) capture_step(e);
    }
    CK(cudaGetLastError());
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- caller-supplied evaluator
extern "C" int b200_ext_capacity(b200_engine *e, int32_t *max_rows, int32_t *out_cols) {
    if (!e || !max_rows || !out_cols) return fail(B200_ERR_BAD_ARG, "null argument");
    if (!ext_kind(e)) return fail(B200_ERR_BAD_ARG, "b200_ext_capacity: the engine's eval_kind is not external");
    *max_rows = e->A.G * (e->A.mode == MODE_LP ? 7 : 1);   // external_game: Vanilla, one leaf per game
    *out_cols = e->A.mode == MODE_DIST ? e->A.dist_bins : 2;
    return B200_OK;
}

// The first half of one simulation step (the same code as b200_run_sims'), then this step's requests in (game, slot) order as boards
// (external) or the leaf games in game order as packed records (external_game).
extern "C" int b200_ext_step_begin(b200_engine *e, void *boards_dev, int board_dtype, int32_t *ids_dev, int32_t *n_rows) {
    if (!e || !boards_dev || !n_rows || (board_dtype != B200_BOARD_INT8 && board_dtype != B200_BOARD_F32 && board_dtype != B200_BOARD_RECORD))
        return fail(B200_ERR_BAD_ARG, "bad argument (boards_dev and n_rows non-NULL, board_dtype B200_BOARD_INT8, B200_BOARD_F32 or B200_BOARD_RECORD)");
    if (!ext_kind(e)) return fail(B200_ERR_BAD_ARG, "b200_ext_step_begin: the engine's eval_kind is not external (use b200_run_sims)");
    if (ext_game_kind(e) && board_dtype != B200_BOARD_RECORD)
        return fail(B200_ERR_BAD_ARG, "b200_ext_step_begin: an external_game engine hands out leaf games: board_dtype B200_BOARD_RECORD");
    if (!ext_game_kind(e) && board_dtype == B200_BOARD_RECORD)
        return fail(B200_ERR_BAD_ARG, "b200_ext_step_begin: an external engine hands out boards: board_dtype B200_BOARD_INT8 or B200_BOARD_F32 "
                                      "(B200_BOARD_RECORD is eval_kind external_game's)");
    if (ext_game_kind(e) && ((uintptr_t)boards_dev & 15))
        return fail(B200_ERR_BAD_ARG, "b200_ext_step_begin: the record buffer must be 16-byte aligned");
    if (e->ext_open) return fail(B200_ERR_BAD_ARG, "b200_ext_step_begin: a step is already open; finish it with b200_ext_step_end");
    CK(cudaSetDevice(e->cfg.device));
    const Arena &A = e->A;
    int rc = step_select(e);
    if (rc) return rc;
    {
        PhaseTimer t(e, PH_MISC);
        const int grid = e->n_sm * 4;
        if (ext_game_kind(e)) {
            k_ext_leaf_order<<<1, EXT_ORDER_THREADS, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n);
            k_ext_leaf_records<<<grid, 256, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n, (uint32_t *)boards_dev, ids_dev);
        } else {
            k_ext_order<<<1, EXT_ORDER_THREADS, 0, e->stream>>>(A, e->d_ext_mark, e->d_ext_rows, e->d_ext_n);
            if (board_dtype == B200_BOARD_INT8) k_ext_boards<int8_t><<<grid, 256, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n, (int8_t *)boards_dev, ids_dev);
            else k_ext_boards<float><<<grid, 256, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n, (float *)boards_dev, ids_dev);
        }
    }
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(&e->ext_rows, e->d_ext_n, sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->ext_open = true;
    *n_rows = e->ext_rows;
    return B200_OK;
}

// The caller's outputs into the evaluator slots, then the backup: the second half of the step b200_ext_step_begin opened.  Asynchronous.
extern "C" int b200_ext_step_end(b200_engine *e, const float *out_dev) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    if (!ext_kind(e)) return fail(B200_ERR_BAD_ARG, "b200_ext_step_end: the engine's eval_kind is not external");
    if (!e->ext_open) return fail(B200_ERR_BAD_ARG, "b200_ext_step_end: no step is open (call b200_ext_step_begin first)");
    if (!out_dev && e->ext_rows > 0) return fail(B200_ERR_BAD_ARG, "b200_ext_step_end: out_dev is NULL");
    CK(cudaSetDevice(e->cfg.device));
    const Arena &A = e->A;
    if (e->ext_rows > 0) {
        PhaseTimer t(e, PH_MISC);
        const int cols = A.mode == MODE_DIST ? A.dist_bins : 2;
        const long long work = ext_game_kind(e) ? e->ext_rows : (long long)e->ext_rows * cols;
        const int grid = (int)std::min<long long>((work + 255) / 256, (long long)e->n_sm * 4);
        if (ext_game_kind(e)) k_ext_leaf_scatter<<<grid, 256, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n, out_dev);
        else k_ext_scatter<<<grid, 256, 0, e->stream>>>(A, e->d_ext_rows, e->d_ext_n, out_dev, cols);
    }
    step_backup(e);
    CK(cudaGetLastError());
    e->ext_open = false;
    return B200_OK;
}

extern "C" int b200_get_stats(b200_engine *e, float *stats, int32_t *action) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    CK(cudaSetDevice(e->cfg.device));
    {
        PhaseTimer t(e, PH_MISC);
        k_root_stats<<<(e->A.G + 127) / 128, 128, 0, e->stream>>>(e->A, e->d_stats, e->d_action);
    }
    CK(cudaGetLastError());
    if (stats) CK(cudaMemcpyAsync(stats, e->d_stats, (size_t)e->A.G * 21 * 4, cudaMemcpyDeviceToHost, e->stream));
    if (action) CK(cudaMemcpyAsync(action, e->d_action, (size_t)e->A.G * 4, cudaMemcpyDeviceToHost, e->stream));
    return check_status(e);
}

extern "C" int b200_env_step(b200_engine *e, const int32_t *actions) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    REFUSE_IF_OPEN(e, "b200_env_step");
    CK(cudaSetDevice(e->cfg.device));
    if (actions) CK(cudaMemcpyAsync(e->d_action, actions, (size_t)e->A.G * 4, cudaMemcpyHostToDevice, e->stream));
    {
        PhaseTimer t(e, PH_MISC);
        k_env_step<<<(e->A.G + 127) / 128, 128, 0, e->stream>>>(e->A.cur, e->d_action, e->A.G);
    }
    CK(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_play_move(b200_engine *e, int sims, int auto_reset, int32_t *actions_out, float *stats_out) {
    if (e) REFUSE_IF_EXT(e, "b200_play_move");
    int rc = b200_run_sims(e, sims);
    if (rc) return rc;
    rc = b200_get_stats(e, stats_out, actions_out);
    if (rc) return rc;
    rc = b200_env_step(e, nullptr);
    if (rc) return rc;
    rc = b200_update_root(e, auto_reset);
    if (rc) return rc;
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// The episodes that ended (and were reset) in the update_root calls since the last drain: out4[i] = {game, score, line_clears, episode},
// at most `cap` rows, count_out = how many ended (may exceed cap: the log holds 4 * n_games rows between drains).  play.py:161-177.
extern "C" int b200_finished_games(b200_engine *e, int32_t *out4, int cap, int32_t *count_out) {
    if (!e || !out4 || cap < 0 || !count_out) return fail(B200_ERR_BAD_ARG, "bad argument");
    CK(cudaSetDevice(e->cfg.device));
    int32_t n = 0;
    CK(cudaMemcpyAsync(&n, e->A.fin_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    *count_out = n;
    int m = n < e->A.fin_cap ? n : e->A.fin_cap;
    if (m > cap) m = cap;
    if (m > 0) CK(cudaMemcpyAsync(out4, e->A.fin_log, (size_t)m * 16, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemsetAsync(e->A.fin_count, 0, 4, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

extern "C" int b200_status(b200_engine *e, int32_t *status) {
    if (!e || !status) return fail(B200_ERR_BAD_ARG, "null argument");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(status, e->A.status, (size_t)e->A.G * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    for (int g = 0; g < e->A.G; ++g)
        status[g] = (status[g] == ST_OK || status[g] == ST_RESET_DONE) ? 0 : (status[g] == ST_ARENA_FULL ? B200_ERR_ARENA_FULL : B200_ERR_TRACE_FULL);
    return B200_OK;
}

extern "C" int b200_counters(b200_engine *e, uint64_t *out16) {
    if (!e || !out16) return fail(B200_ERR_BAD_ARG, "null argument");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(out16, e->A.counters, 16 * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

extern "C" int b200_debug_prof(b200_engine *e, uint64_t *out16) {   // clock64 phase sums of CTA 0 of k_tc_conv (timing mode)
    if (!e || !out16) return fail(B200_ERR_BAD_ARG, "null argument");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(out16, e->A.counters + 16, 16 * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

extern "C" int b200_debug_prof_tree(b200_engine *e, uint64_t *out16) {   // clock64 sums of sampled groups of k_select_expand (timing mode)
    if (!e || !out16) return fail(B200_ERR_BAD_ARG, "null argument");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaMemcpyAsync(out16, e->A.counters + 32, 16 * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

extern "C" int b200_sync(b200_engine *e) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// device-side stopwatch on the engine's own stream (torch.cuda.Event only sees torch's current stream)
extern "C" int b200_timer_start(b200_engine *e) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    CK(cudaSetDevice(e->cfg.device));
    if (!e->t0) { CK(cudaEventCreate(&e->t0)); CK(cudaEventCreate(&e->t1)); }
    CK(cudaStreamSynchronize(e->stream));
    CK(cudaEventRecord(e->t0, e->stream));
    return B200_OK;
}
extern "C" int b200_timer_stop(b200_engine *e, float *ms) {
    if (!e || !ms || !e->t0) return fail(B200_ERR_BAD_ARG, "timer not started");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaEventRecord(e->t1, e->stream));
    CK(cudaEventSynchronize(e->t1));
    CK(cudaEventElapsedTime(ms, e->t0, e->t1));
    return B200_OK;
}

extern "C" int b200_set_timing(b200_engine *e, int on) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    flush_timing(e);
    e->timing = on != 0;
    for (int i = 0; i < PH_N; ++i) { e->phase_ms[i] = 0; e->phase_launches[i] = 0; }
    return B200_OK;
}

extern "C" int b200_phase_ms(b200_engine *e, float *ms8, uint64_t *launches8) {
    if (!e) return fail(B200_ERR_BAD_ARG, "null engine");
    flush_timing(e);
    for (int i = 0; i < PH_N; ++i) { if (ms8) ms8[i] = e->phase_ms[i]; if (launches8) launches8[i] = e->phase_launches[i]; }
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- export
extern "C" int b200_export_game(b200_engine *e, int game, int32_t *child, float *score, int32_t *episode, int32_t *n2o,
                                int32_t *visit, float *value, float *variance, uint8_t *obs_end, uint32_t *game_recs,
                                uint32_t *obs_keys, int32_t *root, int32_t *last_trace, int32_t *last_trace_len) {
    if (!e || game < 0 || game >= e->A.G) return fail(B200_ERR_BAD_ARG, "bad game index");
    CK(cudaSetDevice(e->cfg.device));
    const Arena &A = e->A;
    size_t M = A.M;
    std::vector<int32_t> row(M * ROW_WORDS);
    std::vector<int4> stat(M);
    CK(cudaMemcpyAsync(row.data(), A.row + (size_t)game * M * ROW_WORDS, row.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(stat.data(), A.stat + (size_t)game * M, M * sizeof(int4), cudaMemcpyDeviceToHost, e->stream));
    if (game_recs) CK(cudaMemcpyAsync(game_recs, A.rec + (size_t)game * M * REC_WORDS, M * REC_WORDS * 4, cudaMemcpyDeviceToHost, e->stream));
    if (obs_keys) CK(cudaMemcpyAsync(obs_keys, A.key + (size_t)game * M * KEY_WORDS, M * KEY_WORDS * 4, cudaMemcpyDeviceToHost, e->stream));
    if (root) CK(cudaMemcpyAsync(root, A.root + game, 4, cudaMemcpyDeviceToHost, e->stream));
    int32_t tl = 0;
    CK(cudaMemcpyAsync(&tl, A.trace_len + game, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (last_trace_len) *last_trace_len = tl;
    if (last_trace && tl > 0) {
        CK(cudaMemcpyAsync(last_trace, A.trace + (size_t)game * A.trace_max, (size_t)tl * 4, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaStreamSynchronize(e->stream));
    }
    for (size_t i = 0; i < M; ++i) {   // unpack the 96-byte node record into the reference's separate arrays (agent.py:58-88)
        const int32_t *r = &row[i * ROW_WORDS];
        if (child) for (int a = 0; a < 7; ++a) child[i * 7 + a] = r[a];
        if (episode) episode[i] = r[7];
        if (n2o) n2o[i] = r[15];
        if (score) memcpy(&score[i], &r[23], 4);
        if (visit) visit[i] = stat[i].x;
        if (value) memcpy(&value[i], &stat[i].y, 4);
        if (variance) memcpy(&variance[i], &stat[i].z, 4);
        if (obs_end) obs_end[i] = (uint8_t)(stat[i].w != 0);
    }
    return B200_OK;
}

extern "C" int b200_export_dist(b200_engine *e, int game, float *node_stats, float *node_dist) {
    if (!e || game < 0 || game >= e->A.G || !e->A.nstat) return fail(B200_ERR_BAD_ARG, "not a distributional engine / bad game index");
    CK(cudaSetDevice(e->cfg.device));
    size_t M = e->A.M;
    std::vector<float> ns(M * NSTAT_WORDS);
    CK(cudaMemcpyAsync(ns.data(), e->A.nstat + (size_t)game * M * NSTAT_WORDS, ns.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    if (node_dist) CK(cudaMemcpyAsync(node_dist, e->A.ndist + (size_t)game * M * e->A.dist_bins, M * e->A.dist_bins * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (node_stats) for (size_t i = 0; i < M; ++i) for (int j = 0; j < 5; ++j) node_stats[i * 5 + j] = ns[i * NSTAT_WORDS + j];
    return B200_OK;
}

// DistValueSimOnline.get_value of every game at once (k_dist_root_values): out_dev (DEVICE) double[G][2] = {mean, var} of each root's
// distribution, without copying the arenas to the host
extern "C" int b200_dist_root_values_dev(b200_engine *e, double *out_dev) {
    if (!e || !out_dev) return fail(B200_ERR_BAD_ARG, "null argument");
    if (e->A.mode != MODE_DIST || !e->A.ndist) return fail(B200_ERR_BAD_ARG, "b200_dist_root_values_dev needs B200_MODE_DIST");
    CK(cudaSetDevice(e->cfg.device));
    {
        PhaseTimer t(e, PH_MISC);
        k_dist_root_values<<<(e->A.G + 127) / 128, 128, 0, e->stream>>>(e->A, out_dev);
    }
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- standalone value net
__global__ void k_states_to_keys(const int8_t *states, int k, uint32_t *keys, uint2 *req) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    const int8_t *s = states + (size_t)i * 200;
    uint32_t key[KEY_WORDS];
    for (int q = 0; q < KEY_WORDS; ++q) key[q] = 0;
    uint32_t cells = 0; int n = 0;
    for (int c = 0; c < 200; ++c) {
        int r = c / 10, x = c % 10;
        if (s[c] > 0) key[r >> 1] |= 1u << ((r & 1) * 16 + x);
        else if (s[c] < 0 && n < 4) { cells |= (uint32_t)c << (8 * n); ++n; }
    }
    for (; n < 4; ++n) cells |= 0xffu << (8 * n);   // fewer than four -1 cells: no such cell index (255)
    key[10] = cells;
    for (int q = 0; q < KEY_WORDS; ++q) keys[(size_t)i * KEY_WORDS + q] = key[q];
    // every standalone request gets its own output slot: game = i/8, slot = i%8 -> eval_out[i]
    req[i] = make_uint2((uint32_t)(i >> 3), (uint32_t)i | ((uint32_t)(i & 7) << 28));
}

static int valuenet_forward(b200_engine *e, const int8_t *states, int k, float *v, float *var, uint8_t *dbg, float *dbg_fc) {
    if (!e || !states || !v || !var || k < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (k >= (1 << 28)) return fail(B200_ERR_BAD_ARG, "k too large");
    CK(cudaSetDevice(e->cfg.device));
    int8_t *d_states = nullptr; uint32_t *d_keys = nullptr; uint2 *d_req = nullptr; int32_t *d_n = nullptr; float2 *d_out = nullptr;
    size_t kp = ((size_t)k + 7) & ~(size_t)7;
    Scratch tmp;
    CK(tmp.get(&d_states, (size_t)k * 200)); CK(tmp.get(&d_keys, kp * KEY_WORDS * 4)); CK(tmp.get(&d_req, kp * 8));
    CK(tmp.get(&d_n, 4)); CK(tmp.get(&d_out, kp * 8));
    CK(cudaMemcpyAsync(d_states, states, (size_t)k * 200, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d_n, &k, 4, cudaMemcpyHostToDevice, e->stream));
    k_states_to_keys<<<(k + 127) / 128, 128, 0, e->stream>>>(d_states, k, d_keys, d_req);
    // keys are addressed as keys[(game * M + obs)]: with game = i/8 we pass M = 0 so that only obs (= i) indexes
    int rc = launch_net(e, d_req, d_n, d_keys, 0, d_out, kp, dbg, dbg_fc);
    if (rc == B200_OK) {
        std::vector<float2> h(k);
        cudaError_t ce = cudaMemcpyAsync(h.data(), d_out, (size_t)k * 8, cudaMemcpyDeviceToHost, e->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
        if (ce != cudaSuccess) rc = fail(B200_ERR_CUDA, cudaGetErrorString(ce));
        else for (int i = 0; i < k; ++i) { v[i] = h[i].x; var[i] = h[i].y; }
    }
    cudaStreamSynchronize(e->stream);
    return rc;
}
extern "C" int b200_valuenet_forward(b200_engine *e, const int8_t *states, int k, float *v, float *var) {
    if (e) REFUSE_IF_EXT(e, "b200_valuenet_forward");
    return valuenet_forward(e, states, k, v, var, nullptr, nullptr);
}

// development / test aid: the conv stack's output (flatten input of fc1) in torch order c*56 + y*4 + x, for either path
extern "C" int b200_debug_act3(b200_engine *e, const int8_t *states, int k, float *out) {
    if (e) REFUSE_IF_EXT(e, "b200_debug_act3");
    if (!e || !states || !out || k < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    std::vector<float> v(k), var(k);
    int rc = b200_valuenet_forward(e, states, k, v.data(), var.data());   // leaves act3 of these k boards in the scratch buffers
    if (rc) return rc;
    if (tc_net(e)) {
        TcState *st = (TcState *)e->tc_state;
        const int planes = e->cfg.eval_kind == B200_EVAL_NET_FP16 ? 1 : 2;   // net_fp16 writes the first term only
        size_t bytes = (size_t)2 * st->tiles * ACT3_KCHUNKS * 2048;
        std::vector<uint8_t> h(bytes);
        CK(cudaMemcpy(h.data(), st->d_act3, bytes, cudaMemcpyDeviceToHost));
        for (int r = 0; r < k; ++r)
            for (int kp = 0; kp < 1792; ++kp) {
                int p = kp >> 5, c = kp & 31;
                float sum = 0.f;
                for (int s = planes - 1; s >= 0; --s) {
                    size_t off = ((((size_t)s * st->tiles + (r >> 7)) * ACT3_KCHUNKS + (kp >> 3)) * 128 + (r & 127)) * 16 + (kp & 7) * 2;
                    uint16_t hb; memcpy(&hb, &h[off], 2);
                    sum += host_half_f(hb);
                }
                out[(size_t)r * 1792 + c * 56 + p] = sum / TC_SCALE_A;
            }
        return B200_OK;
    }
    std::vector<float> h((size_t)k * 1792);
    CK(cudaMemcpy(h.data(), e->d_act3, h.size() * 4, cudaMemcpyDeviceToHost));
    for (int r = 0; r < k; ++r)
        for (int y = 0; y < 14; ++y)
            for (int c = 0; c < 32; ++c)
                for (int x = 0; x < 4; ++x) out[(size_t)r * 1792 + c * 56 + y * 4 + x] = h[(size_t)r * 1792 + (y * 32 + c) * 4 + x];
    return B200_OK;
}

// development / test aid: the distributional conv stack's output (flatten input of fc1) in torch order c*64 + y*4 + x, read back from the
// tensor-core kernels' act2 (net_tc: both fp16 terms, dist_fp16: the one it writes)
extern "C" int b200_debug_dist_act2(b200_engine *e, const int8_t *states, int k, float *out) {
    if (e) REFUSE_IF_EXT(e, "b200_debug_dist_act2");
    if (!e || !states || !out || k < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (!dn_tc_net(e)) return fail(B200_ERR_BAD_ARG, "b200_debug_dist_act2 reads the tensor-core distributional network: eval_kind net_tc or dist_fp16");
    if (!e->have_dist_weights) return fail(B200_ERR_NO_WEIGHTS, "b200_load_dist_weights was not called");
    std::vector<float> dist((size_t)k * e->DW.atoms);
    int rc = b200_distnet_forward(e, states, k, e->DW.atoms, dist.data());   // leaves act2 of these k boards in the scratch buffer
    if (rc) return rc;
    DnTcState *st = (DnTcState *)e->dn_tc_state;
    const int planes = e->cfg.eval_kind == B200_EVAL_DIST_FP16 ? 1 : 2;
    size_t bytes = (size_t)2 * st->tiles * DACT2_KCHUNKS * 2048;
    std::vector<uint8_t> h(bytes);
    CK(cudaMemcpy(h.data(), st->d_act2, bytes, cudaMemcpyDeviceToHost));
    for (int r = 0; r < k; ++r)
        for (int kp = 0; kp < 2048; ++kp) {
            int p = kp >> 5, c = kp & 31;
            float sum = 0.f;
            for (int s = planes - 1; s >= 0; --s) {
                size_t off = ((((size_t)s * st->tiles + (r >> 7)) * DACT2_KCHUNKS + (kp >> 3)) * 128 + (r & 127)) * 16 + (kp & 7) * 2;
                uint16_t hb; memcpy(&hb, &h[off], 2);
                sum += host_half_f(hb);
            }
            out[(size_t)r * 2048 + c * 64 + p] = sum / TC_SCALE_A;
        }
    return B200_OK;
}

// development / test aid: every layer of the tensor-core networks exactly as the next layer reads it, and fc1's fp32 accumulator, from one
// forward pass that runs the DBG instantiations of the conv kernel (which also copies the shared-memory activations out) and of the fc
// kernel (which also writes the accumulator out)
extern "C" int b200_debug_tc_acts(b200_engine *e, int dist, const int8_t *states, int k, int layer, float *out) {
    if (e) REFUSE_IF_EXT(e, "b200_debug_tc_acts");
    if (!e || !states || !out || k < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (dist ? !dn_tc_net(e) : !tc_net(e))
        return fail(B200_ERR_BAD_ARG, "b200_debug_tc_acts reads the tensor-core networks: eval_kind net_tc, net_fp16 (value) or dist_fp16 (distributional)");
    if (layer < 0 || layer > (dist ? 3 : 4)) return fail(B200_ERR_BAD_ARG, "layer out of range");
    if (dist ? !e->have_dist_weights : !e->have_weights) return fail(B200_ERR_NO_WEIGHTS, "no weights loaded for this network");
    const int nt = (e->cfg.eval_kind == B200_EVAL_NET_FP16 || e->cfg.eval_kind == B200_EVAL_DIST_FP16) ? 1 : 2;
    const size_t slot = dist ? TDC_ASLOT : TCC_DBG_BYTES;
    const int n_fc1 = dist ? 128 : 256;
    uint8_t *d_dbg = nullptr;
    float *d_fc = nullptr;
    Scratch tmp;
    CK(tmp.get(&d_dbg, (size_t)k * slot));
    CK(tmp.get(&d_fc, (size_t)k * n_fc1 * 4));
    std::vector<float> o0((size_t)k * (dist ? e->DW.atoms : 2));
    int rc;
    if (dist) rc = distnet_forward(e, states, k, e->DW.atoms, o0.data(), d_dbg, d_fc);
    else {
        std::vector<float> v(k), var(k);
        rc = valuenet_forward(e, states, k, v.data(), var.data(), d_dbg, d_fc);
        for (int r = 0; r < k; ++r) { o0[2 * r] = v[r]; o0[2 * r + 1] = var[r]; }
    }
    if (rc) return rc;
    if (layer == 0) { memcpy(out, o0.data(), o0.size() * 4); return B200_OK; }
    if (layer == (dist ? 3 : 4)) {                               // fc1's accumulator: out[k][n_fc1], as the fc kernel's DBG instantiation wrote it
        CK(cudaMemcpy(out, d_fc, (size_t)k * n_fc1 * 4, cudaMemcpyDeviceToHost));
        return B200_OK;
    }
    // out[k][nt][32][H][W]: fp16 term s of channel c at (y, x), divided by TC_SCALE_A
    int H, Wd;
    std::vector<uint8_t> h;
    std::function<size_t(int, int, int, int, int)> off;
    if (layer == (dist ? 2 : 3)) {                               // the conv stack's output: in HBM, the fc kernel's tile layout
        const uint8_t *src; size_t tiles; int kch;
        if (dist) { DnTcState *st = (DnTcState *)e->dn_tc_state; src = st->d_act2; tiles = st->tiles; kch = DACT2_KCHUNKS; H = 16; Wd = 4; }
        else { TcState *st = (TcState *)e->tc_state; src = st->d_act3; tiles = st->tiles; kch = ACT3_KCHUNKS; H = 14; Wd = 4; }
        h.resize((size_t)2 * tiles * kch * 2048);
        CK(cudaMemcpy(h.data(), src, h.size(), cudaMemcpyDeviceToHost));
        off = [=](int r, int s, int c, int y, int x) {
            const int kp = (y * 4 + x) * 32 + c;
            return ((((size_t)s * tiles + (r >> 7)) * kch + (kp >> 3)) * 128 + (r & 127)) * 16 + (kp & 7) * 2;
        };
    } else {                                                     // a shared-memory slot copied by the DBG kernel
        h.resize((size_t)k * slot);
        CK(cudaMemcpy(h.data(), d_dbg, h.size(), cudaMemcpyDeviceToHost));
        if (dist) {                                              // act1: [term][chunk 4][152 rows][16 B], row y*8 + x
            H = 19; Wd = 7;
            off = [=](int r, int s, int c, int y, int x) { return r * slot + (size_t)s * 4 * TDC_R * 16 + ((c >> 3) * TDC_R + y * 8 + x) * 16 + (c & 7) * 2; };
        } else if (layer == 1) {                                 // act1: [term][chunk 4][144 rows][16 B], row y*8 + x
            H = 18; Wd = 8;
            off = [=](int r, int s, int c, int y, int x) { return r * slot + (size_t)s * 4 * TCC_R * 16 + ((c >> 3) * TCC_R + y * 8 + x) * 16 + (c & 7) * 2; };
        } else {                                                 // act2: [term, stride TCC_A2SPLIT][chunk 4][98 rows][16 B], row x*16 + y
            H = 16; Wd = 6;
            off = [=](int r, int s, int c, int y, int x) {
                return r * slot + TCC_ASLOT + (size_t)s * TCC_A2SPLIT + ((c >> 3) * TCC_R2 + x * 16 + y) * 16 + (c & 7) * 2;
            };
        }
    }
    for (int r = 0; r < k; ++r)
        for (int s = 0; s < nt; ++s)
            for (int c = 0; c < 32; ++c)
                for (int y = 0; y < H; ++y)
                    for (int x = 0; x < Wd; ++x) {
                        uint16_t hb; memcpy(&hb, &h[off(r, s, c, y, x)], 2);
                        out[((((size_t)r * nt + s) * 32 + c) * H + y) * Wd + x] = host_half_f(hb) / TC_SCALE_A;
                    }
    return B200_OK;
}

// development / test aid: every stage of the fp32 CUDA-core networks (eval_kind net) exactly as the kernels computed it, from one forward
// pass that runs the DBG instantiations k_vn_conv_dbg / k_vn_fc_dbg or k_dn_conv_dbg / k_dn_fc_dbg
extern "C" int b200_debug_net_acts(b200_engine *e, int dist, const int8_t *states, int k, int layer, float *out) {
    if (e) REFUSE_IF_EXT(e, "b200_debug_net_acts");
    if (!e || !states || !out || k < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (e->cfg.eval_kind != B200_EVAL_NET) return fail(B200_ERR_BAD_ARG, "b200_debug_net_acts reads the fp32 CUDA-core networks: eval_kind net");
    if (dist != 0 && dist != 1) return fail(B200_ERR_BAD_ARG, "dist must be 0 (value network) or 1 (distributional network)");
    if (layer < 0 || layer > 4) return fail(B200_ERR_BAD_ARG, "layer out of range");
    if (dist ? !e->have_dist_weights : !e->have_weights) return fail(B200_ERR_NO_WEIGHTS, "no weights loaded for this network");
    const int atoms = e->DW.atoms;
    const size_t slot = dist ? DN_DBG_A1 : VN_DBG_FLOATS, n_fc1 = dist ? 128 : 256;
    float *d_dbg = nullptr, *d_fc = nullptr, *d_lg = nullptr;
    Scratch tmp;
    CK(tmp.get(&d_dbg, (size_t)k * slot * 4));
    CK(tmp.get(&d_fc, (size_t)k * n_fc1 * 4));
    if (dist) CK(tmp.get(&d_lg, (size_t)k * atoms * 4));
    std::vector<float> o0((size_t)k * (dist ? atoms : 2));
    int rc;
    if (dist) rc = distnet_forward(e, states, k, atoms, o0.data(), reinterpret_cast<uint8_t *>(d_dbg), d_fc, d_lg);
    else {
        std::vector<float> v(k), var(k);
        rc = valuenet_forward(e, states, k, v.data(), var.data(), reinterpret_cast<uint8_t *>(d_dbg), d_fc);
        for (int r = 0; r < k; ++r) { o0[2 * r] = v[r]; o0[2 * r + 1] = var[r]; }
    }
    if (rc) return rc;
    if (layer == 0) { memcpy(out, o0.data(), o0.size() * 4); return B200_OK; }
    const float *src = nullptr;        // layers already in their output layout: copied as they are
    size_t n = 0;
    if (dist) {
        if (layer == 1) { src = d_dbg; n = (size_t)k * DN_DBG_A1; }                  // act1 [32][19][7]
        else if (layer == 2) { src = e->d_dn_act; n = (size_t)k * 2048; }        // act2 [32][16][4], the production buffer
        else if (layer == 3) { src = d_fc; n = (size_t)k * 128; }                // fc1, bias included, before the LeakyReLU
        else { src = d_lg; n = (size_t)k * atoms; }                              // logits
    } else if (layer == 4) { src = d_fc; n = (size_t)k * 256; }                  // fc1's accumulator, before the bias and the ReLU
    if (src) { CK(cudaMemcpy(out, src, n * 4, cudaMemcpyDeviceToHost)); return B200_OK; }
    if (layer == 3) {                                                            // act3 [32][14][4] from the production buffer
        std::vector<float> h((size_t)k * 1792);
        CK(cudaMemcpy(h.data(), e->d_act3, h.size() * 4, cudaMemcpyDeviceToHost));
        for (int r = 0; r < k; ++r)
            for (int y = 0; y < 14; ++y)
                for (int c = 0; c < 32; ++c)
                    for (int x = 0; x < 4; ++x) out[(size_t)r * 1792 + c * 56 + y * 4 + x] = h[(size_t)r * 1792 + (y * 32 + c) * 4 + x];
        return B200_OK;
    }
    std::vector<float> h((size_t)k * VN_DBG_FLOATS);                             // act1 [32][18][8] | act2 [32][16][6] per board
    CK(cudaMemcpy(h.data(), d_dbg, h.size() * 4, cudaMemcpyDeviceToHost));
    const int off = layer == 1 ? 0 : VN_DBG_A1, len = layer == 1 ? VN_DBG_A1 : VN_DBG_FLOATS - VN_DBG_A1;
    for (int r = 0; r < k; ++r) memcpy(out + (size_t)r * len, h.data() + (size_t)r * VN_DBG_FLOATS + off, (size_t)len * 4);
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- standalone env
static int env_stream_op(uint32_t *recs, const int32_t *actions, int8_t *state_out, int n) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    uint32_t *d = nullptr; int32_t *da = nullptr; int8_t *ds = nullptr;
    Scratch tmp;
    CK(tmp.get(&d, (size_t)n * REC_WORDS * 4));
    CK(cudaMemcpy(d, recs, (size_t)n * REC_WORDS * 4, cudaMemcpyHostToDevice));
    if (actions) {
        CK(tmp.get(&da, (size_t)n * 4));
        CK(cudaMemcpy(da, actions, (size_t)n * 4, cudaMemcpyHostToDevice));
        k_env_step<<<(n + 127) / 128, 128>>>(d, da, n);
        CK(cudaGetLastError());
        CK(cudaMemcpy(recs, d, (size_t)n * REC_WORDS * 4, cudaMemcpyDeviceToHost));
    }
    if (state_out) {
        CK(tmp.get(&ds, (size_t)n * 200));
        k_env_state<<<(n + 127) / 128, 128>>>(d, ds, n);
        CK(cudaGetLastError());
        CK(cudaMemcpy(state_out, ds, (size_t)n * 200, cudaMemcpyDeviceToHost));
    }
    return B200_OK;
}

extern "C" int b200_tetris_new(uint32_t *recs, int n, int app, int scoring, int randomizer, const uint32_t *seeds, int reset) {
    if (!recs || n < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    uint32_t *d = nullptr, *ds = nullptr;
    Scratch tmp;
    CK(tmp.get(&d, (size_t)n * REC_WORDS * 4));
    if (reset) CK(cudaMemcpy(d, recs, (size_t)n * REC_WORDS * 4, cudaMemcpyHostToDevice));
    if (seeds && !reset) { CK(tmp.get(&ds, (size_t)n * 4)); CK(cudaMemcpy(ds, seeds, (size_t)n * 4, cudaMemcpyHostToDevice)); }
    k_new_games<<<(n + 127) / 128, 128>>>(d, n, app, scoring, randomizer, ds, reset);
    CK(cudaGetLastError());
    CK(cudaMemcpy(recs, d, (size_t)n * REC_WORDS * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
}

extern "C" int b200_tetris_step(uint32_t *recs, const int32_t *actions, int n) {
    if (!recs || !actions || n < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    return env_stream_op(recs, actions, nullptr, n);
}
extern "C" int b200_tetris_state(const uint32_t *recs, int8_t *out, int n) {
    if (!recs || !out || n < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    return env_stream_op(const_cast<uint32_t *>(recs), nullptr, out, n);
}

// ---------------------------------------------------------------------------------------------------- caller-owned device games
// Tetris.play / getState / random playouts on DEVICE records, asynchronous on the caller's stream (no engine, no copy, no synchronisation).
static int dev_games_arg(const void *recs_dev, int n, const char *fn) {
    if ((!recs_dev && n > 0) || n < 0) return fail(B200_ERR_BAD_ARG, std::string(fn) + ": recs_dev non-NULL and n >= 0");
    if ((uintptr_t)recs_dev & 15) return fail(B200_ERR_BAD_ARG, std::string(fn) + ": recs_dev must be 16-byte aligned");
    return B200_OK;
}

extern "C" int b200_tetris_step_dev(uint32_t *recs_dev, const int32_t *actions_dev, int n, void *stream) {
    if (int rc = dev_games_arg(recs_dev, n, "b200_tetris_step_dev")) return rc;
    if (!actions_dev && n > 0) return fail(B200_ERR_BAD_ARG, "b200_tetris_step_dev: actions_dev is NULL");
    if (n == 0) return B200_OK;
    k_env_step<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(recs_dev, actions_dev, n);
    CK(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_tetris_state_dev(const uint32_t *recs_dev, void *out_dev, int dtype, int n, void *stream) {
    if (int rc = dev_games_arg(recs_dev, n, "b200_tetris_state_dev")) return rc;
    if ((!out_dev && n > 0) || (dtype != B200_BOARD_INT8 && dtype != B200_BOARD_F32))
        return fail(B200_ERR_BAD_ARG, "b200_tetris_state_dev: out_dev non-NULL, dtype B200_BOARD_INT8 or B200_BOARD_F32");
    if (n == 0) return B200_OK;
    const int grid = (n + GAME_STATE_THREADS - 1) / GAME_STATE_THREADS;
    if (dtype == B200_BOARD_INT8) k_game_state<int8_t><<<grid, GAME_STATE_THREADS, 0, (cudaStream_t)stream>>>(recs_dev, (int8_t *)out_dev, n);
    else k_game_state<float><<<grid, GAME_STATE_THREADS, 0, (cudaStream_t)stream>>>(recs_dev, (float *)out_dev, n);
    CK(cudaGetLastError());
    return B200_OK;
}

extern "C" int b200_tetris_playout_dev(uint32_t *recs_dev, uint32_t *rng_dev, int n, int n_actions, int max_steps, int32_t *steps_dev, void *stream) {
    if (int rc = dev_games_arg(recs_dev, n, "b200_tetris_playout_dev")) return rc;
    if ((!rng_dev && n > 0) || n_actions < 1 || n_actions > 8 || max_steps < 0)
        return fail(B200_ERR_BAD_ARG, "b200_tetris_playout_dev: rng_dev non-NULL, 1 <= n_actions <= 8, max_steps >= 0");
    if (n == 0) return B200_OK;
    k_game_playout<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(recs_dev, rng_dev, n, n_actions, max_steps, steps_dev);
    CK(cudaGetLastError());
    return B200_OK;
}

// test aids on trees given in the reference's layout (agents/agent.py:58-88): every child id and observation id within [0, M)
static bool ref_tree_in_range(int M, const int32_t *child, const int32_t *n_to_o) {
    for (int i = 0; i < M; ++i)
        if (n_to_o[i] < 0 || n_to_o[i] >= M) return false;
    for (int i = 0; i < M * 7; ++i)
        if (child[i] < 0 || child[i] >= M) return false;
    return true;
}

// the rows (c / o / s from child, n_to_o, score; the link words are left to finish_expansion, k_debug_link_rows) and the statistics
// (visit / value / variance / end per observation) of such a tree, as the engine holds them
static void ref_tree_rows(int M, const int32_t *child, const int32_t *n_to_o, const float *score, const int32_t *visit, const float *value,
                          const float *variance, const uint8_t *end, std::vector<int32_t> &row, std::vector<int4> &st) {
    row.assign((size_t)M * ROW_WORDS, 0);
    st.resize(M);
    for (int i = 0; i < M; ++i) {
        int32_t *r = &row[(size_t)i * ROW_WORDS];
        for (int a = 0; a < 7; ++a) { const int c = child[(size_t)i * 7 + a]; r[a] = c; r[8 + a] = n_to_o[c]; memcpy(&r[16 + a], &score[c], 4); }
        r[15] = n_to_o[i]; memcpy(&r[23], &score[i], 4);
        int4 s; s.x = visit[i]; memcpy(&s.y, &value[i], 4); memcpy(&s.z, &variance[i], 4); s.w = end[i] != 0;
        st[i] = s;
    }
}

// test aid: game `game` of an engine (mode lp, single or vanilla) as expansions would have left the tree given in the reference's layout:
// the rows with the link words of the production finish_expansion, the statistics, the root, the game's check_low stream srng = rng_state
// (non-zero), status ST_OK, an empty path cache, and node records whose game-over bit is set exactly on the nodes without children.  Every
// walk of b200_run_sims then ends at a terminal leaf: the production walk (k_select_expand) and the terminal backup (k_backup) run on the
// given statistics with no expansion, evaluation or collection.  Nodes >= M of the game keep what they held (no walk reaches them).
extern "C" int b200_debug_load_tree(b200_engine *e, int game, int M, const int32_t *child, const int32_t *n_to_o, const float *score,
                                    const int32_t *visit, const float *value, const float *variance, const uint8_t *end, int root,
                                    uint32_t rng_state) {
    if (!e || !child || !n_to_o || !score || !visit || !value || !variance || !end) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_OPEN(e, "b200_debug_load_tree");
    Arena &A = e->A;
    if (A.mode != MODE_LP && A.mode != MODE_SINGLE && A.mode != MODE_VANILLA) return fail(B200_ERR_BAD_ARG, "b200_debug_load_tree needs an engine of mode lp, single or vanilla");
    if (game < 0 || game >= A.G || M < 2 || M > A.M || root < 1 || root >= M || rng_state == 0u)
        return fail(B200_ERR_BAD_ARG, "need 0 <= game < n_games, 2 <= M <= max_nodes, 1 <= root < M and rng_state != 0");
    if (!ref_tree_in_range(M, child, n_to_o)) return fail(B200_ERR_BAD_ARG, "child or n_to_o out of range");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaStreamSynchronize(e->stream));
    std::vector<int32_t> row;
    std::vector<int4> st;
    ref_tree_rows(M, child, n_to_o, score, visit, value, variance, end, row, st);
    std::vector<uint32_t> rec((size_t)M * REC_WORDS, 0u);
    for (int i = 0; i < M; ++i) {
        bool leaf = true;
        for (int a = 0; a < 7; ++a) leaf = leaf && child[(size_t)i * 7 + a] == 0;
        rec[(size_t)i * REC_WORDS + 10] = leaf ? 1u << 21 : 0u;        // the game-over bit k_select_expand reads from the leaf's record
    }
    const int32_t zero = 0, st_ok = ST_OK;
    CK(cudaMemcpyAsync(A.row + (size_t)game * A.M * ROW_WORDS, row.data(), row.size() * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.stat + (size_t)game * A.M, st.data(), (size_t)M * sizeof(int4), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.rec + (size_t)game * A.M * REC_WORDS, rec.data(), rec.size() * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.root + game, &root, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.srng + game, &rng_state, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.status + game, &st_ok, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.pending + game, &zero, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.trace_len + game, &zero, 4, cudaMemcpyHostToDevice, e->stream));
    if (A.pc) CK(cudaMemcpyAsync(A.pc_len + game, &zero, 4, cudaMemcpyHostToDevice, e->stream));
    k_debug_link_rows<<<(M + 15) / 16, 128, 0, e->stream>>>(A, game, M);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// test aid: a game's check_low stream state and its path cache's valid length (0 with the cache off)
extern "C" int b200_debug_game_state(b200_engine *e, int game, uint32_t *rng_state, int32_t *pc_len) {
    if (!e || !rng_state || !pc_len || game < 0 || game >= e->A.G) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_OPEN(e, "b200_debug_game_state");
    CK(cudaSetDevice(e->cfg.device));
    *pc_len = 0;
    CK(cudaMemcpyAsync(rng_state, e->A.srng + game, 4, cudaMemcpyDeviceToHost, e->stream));
    if (e->A.pc) CK(cudaMemcpyAsync(pc_len, e->A.pc_len + game, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// development / test aid: the production k_backup (through step_backup, the launch run_sims uses) on a tree given in the reference's layout
// (agents/agent.py:58-88), on game 0 of a one-game engine.  The game's row (c / o / s from child, n_to_o, score; the link words by
// finish_expansion), stat (visit / value / variance / end per observation), trace, trace_meta (own observation | pick << 28, own score; the
// pick = the first slot holding the next level's observation), leaf_kind and the evaluator outputs (eval_out[8][2] per slot, rollout_val)
// are written as a walk and an evaluation would leave them; visit / value / variance come back in place.  With the path cache on, pc_len
// (in: the entries the walk left valid, <= D - 1 after an expansion, <= D at a terminal leaf) is filled from the pre-backup arena by the
// walk's own store (k_debug_pc_fill) and returned with the entries: pc_own[D][4], pc_sib[D][8], pc_ent[D][8][4] ({link word, val, visit,
// root}; slot 7 {0, own score, own observation, node}), pc_var[D][8].
extern "C" int b200_debug_backup(b200_engine *e, int M, const int32_t *child, const int32_t *n_to_o, const float *score, int32_t *visit,
                                 float *value, float *variance, const uint8_t *end, const int32_t *trace, int D, int leaf_kind,
                                 const float *eval_out, float rollout_val, int32_t *pc_len, int32_t *pc_own, uint16_t *pc_sib,
                                 int32_t *pc_ent, int32_t *pc_var) {
    if (!e || !child || !n_to_o || !score || !visit || !value || !variance || !end || !trace || !eval_out) return fail(B200_ERR_BAD_ARG, "bad argument");
    REFUSE_IF_OPEN(e, "b200_debug_backup");
    Arena &A = e->A;
    if (A.G != 1 || (A.mode != MODE_LP && A.mode != MODE_SINGLE && A.mode != MODE_VANILLA)) return fail(B200_ERR_BAD_ARG, "b200_debug_backup needs a one-game engine of mode lp, single or vanilla");
    if (M < 2 || M > A.M || D < 1 || D > A.trace_max) return fail(B200_ERR_BAD_ARG, "need 2 <= M <= max_nodes and 1 <= D <= trace_max");
    if (leaf_kind != LEAF_TERMINAL && leaf_kind != LEAF_EXPANDED) return fail(B200_ERR_BAD_ARG, "leaf_kind: 0 terminal or 1 expanded");
    if (!A.pc != !pc_len || (pc_len && (!pc_own || !pc_sib || !pc_ent || !pc_var)))
        return fail(B200_ERR_BAD_ARG, "pc_len and the entry buffers are given exactly when the path cache is on");
    if (pc_len && (*pc_len < 0 || *pc_len > (leaf_kind == LEAF_EXPANDED ? D - 1 : D))) return fail(B200_ERR_BAD_ARG, "pc_len beyond what a walk leaves valid");
    if (!ref_tree_in_range(M, child, n_to_o)) return fail(B200_ERR_BAD_ARG, "child or n_to_o out of range");
    for (int d = 0; d < D; ++d)
        if (trace[d] < 1 || trace[d] >= M) return fail(B200_ERR_BAD_ARG, "trace entry out of range");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaStreamSynchronize(e->stream));
    std::vector<int32_t> row;
    std::vector<int4> st;
    ref_tree_rows(M, child, n_to_o, score, visit, value, variance, end, row, st);
    std::vector<int2> meta(D);
    for (int d = 0; d < D; ++d) {
        const int32_t *r = &row[(size_t)trace[d] * ROW_WORDS];
        int pick = 0;
        if (d + 1 < D) {
            const int want = n_to_o[trace[d + 1]];
            pick = 7;
            for (int a = 0; a < 7 && pick == 7; ++a) if (r[a] != 0 && r[8 + a] == want) pick = a;
        }
        meta[d] = make_int2(r[15] | (pick << 28), r[23]);
    }
    const int32_t st_ok = ST_OK;
    CK(cudaMemcpyAsync(A.row, row.data(), row.size() * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.stat, st.data(), (size_t)M * sizeof(int4), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.trace, trace, (size_t)D * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.trace_meta, meta.data(), (size_t)D * sizeof(int2), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.trace_len, &D, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.leaf_kind, &leaf_kind, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.status, &st_ok, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.eval_out, eval_out, 8 * sizeof(float2), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(A.rollout_val, &rollout_val, 4, cudaMemcpyHostToDevice, e->stream));
    k_debug_link_rows<<<(M + 15) / 16, 128, 0, e->stream>>>(A, 0, M);
    if (pc_len) {
        k_debug_pc_fill<<<1, 8, 0, e->stream>>>(A, 0, *pc_len, D);
        CK(cudaMemcpyAsync(A.pc_len, pc_len, 4, cudaMemcpyHostToDevice, e->stream));
    }
    step_backup(e);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(st.data(), A.stat, (size_t)M * sizeof(int4), cudaMemcpyDeviceToHost, e->stream));
    std::vector<int4> own, ent((size_t)8 * A.trace_max);
    std::vector<uint4> sib;
    std::vector<int32_t> pvar((size_t)8 * A.trace_max);
    if (pc_len) {
        own.resize(D); sib.resize(D);
        CK(cudaMemcpyAsync(pc_len, A.pc_len, 4, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(own.data(), A.pc_own, (size_t)D * sizeof(int4), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(sib.data(), A.pc_sib, (size_t)D * sizeof(uint4), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(ent.data(), A.pc, ent.size() * sizeof(int4), cudaMemcpyDeviceToHost, e->stream));
        CK(cudaMemcpyAsync(pvar.data(), A.pc_var, pvar.size() * 4, cudaMemcpyDeviceToHost, e->stream));
    }
    CK(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < M; ++i) { visit[i] = st[i].x; memcpy(&value[i], &st[i].y, 4); memcpy(&variance[i], &st[i].z, 4); }
    if (pc_len) {
        for (int d = 0; d < D; ++d) {
            pc_own[4 * d] = own[d].x; pc_own[4 * d + 1] = own[d].y; pc_own[4 * d + 2] = own[d].z; pc_own[4 * d + 3] = own[d].w;
            memcpy(pc_sib + 8 * d, &sib[d], 16);
            for (int a = 0; a < 8; ++a) {   // slot-major [8][trace_max] on the device
                const int4 v = ent[(size_t)a * A.trace_max + d];
                int32_t *o = pc_ent + ((size_t)d * 8 + a) * 4;
                o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
                pc_var[(size_t)d * 8 + a] = pvar[(size_t)a * A.trace_max + d];
            }
        }
    }
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- core twins
struct TwinBufs {
    int32_t *child = nullptr, *visit = nullptr, *n2o = nullptr, *trace = nullptr, *out = nullptr;
    float *value = nullptr, *variance = nullptr, *score = nullptr, *zt = nullptr;
    uint32_t *rng = nullptr;
    std::vector<void *> all;
    ~TwinBufs() { for (void *p : all) cudaFree(p); }
    template <typename T> int up(T **d, const T *h, size_t n) {
        if (cudaMalloc((void **)d, (n ? n : 1) * sizeof(T)) != cudaSuccess) return 1;
        all.push_back(*d);
        if (h && n) return cudaMemcpy(*d, h, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess;
        return cudaMemset(*d, 0, (n ? n : 1) * sizeof(T)) != cudaSuccess;
    }
};

static int twin_arena(TwinBufs &b, Arena &A) {
    memset(&A, 0, sizeof(A));
    std::vector<float> h(ZTABLE_N);
    const double l2 = log(2.0), l22 = log(22.0), l41 = log(41.0);
    for (int n = 0; n < ZTABLE_N; ++n) {
        double t = (double)n, alpha = 1 - 1 / t;
        h[n] = (float)(10 * log(1 - log(-log(alpha) / l2) / l22) / l41);
    }
    if (b.up(&b.zt, h.data(), (size_t)ZTABLE_N)) return 1;
    A.ztable = b.zt;
    return 0;
}

#define TW(x) do { if (x) return fail(B200_ERR_CUDA, "twin: device allocation/copy failed"); } while (0)

extern "C" int b200_select_trace_obs(int index, const int32_t *child, const int32_t *visit, const float *value,
                                     const float *variance, const float *score, const int32_t *n_to_o, int M, int low,
                                     uint32_t *rng_state, int32_t *trace_out, int max_trace, int32_t *trace_len) {
    if (!child || !visit || !value || !variance || !score || !n_to_o || !trace_out || !trace_len || index < 0 || index >= M)
        return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; Arena A;
    TW(twin_arena(b, A));
    uint32_t seed = rng_state ? *rng_state : 0x2545F491u;
    TW(b.up(&b.child, child, (size_t)M * 7)); TW(b.up(&b.visit, visit, (size_t)M)); TW(b.up(&b.value, value, (size_t)M));
    TW(b.up(&b.variance, variance, (size_t)M)); TW(b.up(&b.score, score, (size_t)M)); TW(b.up(&b.n2o, n_to_o, (size_t)M));
    TW(b.up(&b.trace, (const int32_t *)nullptr, (size_t)max_trace)); TW(b.up(&b.out, (const int32_t *)nullptr, 16)); TW(b.up(&b.rng, &seed, 1));
    TwinArgs t{b.child, b.visit, b.value, b.variance, b.score, b.n2o, b.trace, b.rng, b.out};
    k_twin_select<<<1, 32>>>(A, t, index, low, max_trace);
    CK(cudaGetLastError());
    int32_t out[2];
    CK(cudaMemcpy(out, b.out, 8, cudaMemcpyDeviceToHost));
    if (out[1] != ST_OK) return fail(B200_ERR_TRACE_FULL, "trace longer than max_trace");
    CK(cudaMemcpy(trace_out, b.trace, (size_t)out[0] * 4, cudaMemcpyDeviceToHost));
    if (rng_state) CK(cudaMemcpy(rng_state, b.rng, 4, cudaMemcpyDeviceToHost));
    *trace_len = out[0];
    return B200_OK;
}

extern "C" int b200_get_unique_child_obs(int index, const int32_t *child, const float *score, const int32_t *n_to_o, int M,
                                         int32_t *c_nodes, int32_t *c_obs, int32_t *k_out) {
    if (!child || !score || !n_to_o || !c_nodes || !c_obs || !k_out || index < 0 || index >= M) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; Arena A;
    TW(twin_arena(b, A));
    TW(b.up(&b.child, child, (size_t)M * 7)); TW(b.up(&b.score, score, (size_t)M)); TW(b.up(&b.n2o, n_to_o, (size_t)M));
    TW(b.up(&b.out, (const int32_t *)nullptr, 16));
    TwinArgs t{b.child, nullptr, nullptr, nullptr, b.score, b.n2o, nullptr, nullptr, b.out};
    k_twin_unique<<<1, 32>>>(A, t, index);
    CK(cudaGetLastError());
    int32_t out[16];
    CK(cudaMemcpy(out, b.out, 64, cudaMemcpyDeviceToHost));
    *k_out = out[0];
    for (int i = 0; i < out[0]; ++i) { c_nodes[i] = out[1 + i]; c_obs[i] = out[8 + i]; }
    return B200_OK;
}

static int twin_backup_common(TwinBufs &b, const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                              const int32_t *n_to_o, const float *score, int M) {
    if (b.up(&b.trace, trace, (size_t)D) || b.up(&b.visit, (const int32_t *)visit, (size_t)M) || b.up(&b.value, (const float *)value, (size_t)M) ||
        b.up(&b.variance, (const float *)variance, (size_t)M) || b.up(&b.n2o, n_to_o, (size_t)M) || b.up(&b.score, score, (size_t)M)) return 1;
    return 0;
}
static int twin_backup_fetch(TwinBufs &b, int32_t *visit, float *value, float *variance, int M) {
    if (cudaMemcpy(visit, b.visit, (size_t)M * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    if (cudaMemcpy(value, b.value, (size_t)M * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    if (cudaMemcpy(variance, b.variance, (size_t)M * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
    return 0;
}

extern "C" int b200_backup_trace_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                                     const int32_t *n_to_o, const float *score, int M, double v, double var, double gamma) {
    if (!trace || D < 1 || !visit || !value || !variance || !n_to_o || !score) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; Arena A;
    TW(twin_arena(b, A));
    TW(twin_backup_common(b, trace, D, visit, value, variance, n_to_o, score, M));
    TwinArgs t{nullptr, b.visit, b.value, b.variance, b.score, b.n2o, b.trace, nullptr, nullptr};
    k_twin_backup<<<1, 1>>>(A, t, D, v, var, gamma, 0);
    CK(cudaGetLastError());
    TW(twin_backup_fetch(b, visit, value, variance, M));
    return B200_OK;
}

extern "C" int b200_backup_trace_obs_LP(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                                        const int32_t *n_to_o, const float *score, const uint8_t *end, int M,
                                        const int32_t *c_nodes, const int32_t *c_obs, int k, const float *v, const float *var,
                                        double gamma, int mixture, int averaged) {
    if (!trace || D < 1 || !visit || !value || !variance || !n_to_o || !score || !end || k < 0 || k > 7) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; Arena A;
    TW(twin_arena(b, A));
    TW(twin_backup_common(b, trace, D, visit, value, variance, n_to_o, score, M));
    uint8_t *d_end = nullptr; int32_t *d_cn = nullptr, *d_co = nullptr; float *d_v = nullptr, *d_var = nullptr;
    TW(b.up(&d_end, end, (size_t)M)); TW(b.up(&d_cn, c_nodes, (size_t)k)); TW(b.up(&d_co, c_obs, (size_t)k));
    TW(b.up(&d_v, v, (size_t)k)); TW(b.up(&d_var, var, (size_t)k));
    TwinArgs t{nullptr, b.visit, b.value, b.variance, b.score, b.n2o, b.trace, nullptr, nullptr};
    k_twin_backup_lp<<<1, 1>>>(A, t, D, d_end, d_cn, d_co, k, d_v, d_var, gamma, mixture, averaged);
    CK(cudaGetLastError());
    TW(twin_backup_fetch(b, visit, value, variance, M));
    return B200_OK;
}

// test aid: the walk's z(n) (search_dev.cuh ztab) for n[count]: out[i] as policy_clt's bound coefficient (core.h:93) on the device
extern "C" int b200_debug_ztab(const int32_t *n, int count, float *out) {
    if (!n || !out || count < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; Arena A;
    TW(twin_arena(b, A));
    int32_t *d_n = nullptr; float *d_out = nullptr;
    TW(b.up(&d_n, n, (size_t)count)); TW(b.up(&d_out, (const float *)nullptr, (size_t)count));
    k_debug_ztab<<<256, 256>>>(A, d_n, count, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out, (size_t)count * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
}

extern "C" int b200_get_all_childs(int index, const int32_t *child, int M, uint8_t *mark) {
    if (!child || !mark || index < 0 || index >= M) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b;
    uint8_t *d_mark = nullptr; int32_t *d_q = nullptr;
    TW(b.up(&b.child, child, (size_t)M * 7)); TW(b.up(&d_mark, (const uint8_t *)nullptr, (size_t)M)); TW(b.up(&d_q, (const int32_t *)nullptr, (size_t)M));
    k_twin_all_childs<<<1, 32>>>(b.child, M, index, d_mark, d_q);
    CK(cudaGetLastError());
    CK(cudaMemcpy(mark, d_mark, (size_t)M, cudaMemcpyDeviceToHost));
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- distributional cores (a16)
extern "C" int b200_dist_shift_distribution(const float *dist, int bins, double x, double vmin, double vmax, float *out) {
    if (!dist || !out || bins < 1 || bins > 4096 || !(x >= 0)) return fail(B200_ERR_BAD_ARG, "bad argument");   // x < 0 would index below bin 0
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; float *d_in = nullptr, *d_out = nullptr;
    TW(b.up(&d_in, dist, (size_t)bins)); TW(b.up(&d_out, (const float *)nullptr, (size_t)bins));
    k_dist_shift<<<1, 1>>>(d_in, bins, x, vmin, vmax, d_out);
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out, (size_t)bins * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
}

extern "C" int b200_dist_mean_variance(const float *dist, int bins, double vmin, double vmax, double *mean, double *var) {
    if (!dist || !mean || !var || bins < 1) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; float *d_in = nullptr; double *d_out = nullptr;
    TW(b.up(&d_in, dist, (size_t)bins)); TW(b.up(&d_out, (const double *)nullptr, 2));
    k_dist_mean_variance<<<1, 1>>>(d_in, bins, vmin, vmax, d_out);
    CK(cudaGetLastError());
    double h[2];
    CK(cudaMemcpy(h, d_out, 16, cudaMemcpyDeviceToHost));
    *mean = h[0]; *var = h[1];
    return B200_OK;
}

extern "C" int b200_dist_select_trace(int index, const int32_t *child, const float *node_stats, int M, int low, uint32_t *rng_state,
                                      int32_t *trace_out, int max_trace, int32_t *trace_len) {
    if (!child || !node_stats || !trace_out || !trace_len || index < 0 || index >= M) return fail(B200_ERR_BAD_ARG, "bad argument");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; float *d_ns = nullptr; int32_t *d_len = nullptr;
    uint32_t seed = rng_state ? *rng_state : 0x2545F491u;
    TW(b.up(&b.child, child, (size_t)M * 7)); TW(b.up(&d_ns, node_stats, (size_t)M * 5)); TW(b.up(&b.trace, (const int32_t *)nullptr, (size_t)max_trace));
    TW(b.up(&b.rng, &seed, 1)); TW(b.up(&d_len, (const int32_t *)nullptr, 1));
    k_dist_select<<<1, 1>>>(index, b.child, d_ns, low, b.trace, max_trace, b.rng, d_len);
    CK(cudaGetLastError());
    int32_t n = 0;
    CK(cudaMemcpy(&n, d_len, 4, cudaMemcpyDeviceToHost));
    if (n < 0) return fail(B200_ERR_TRACE_FULL, "trace longer than max_trace");
    CK(cudaMemcpy(trace_out, b.trace, (size_t)n * 4, cudaMemcpyDeviceToHost));
    if (rng_state) CK(cudaMemcpy(rng_state, b.rng, 4, cudaMemcpyDeviceToHost));
    *trace_len = n;
    return B200_OK;
}

extern "C" int b200_dist_backup_trace(const int32_t *trace, int D, float *node_stats, float *node_dist, int M, int bins, double r,
                                      const float *dist, double vmin, double vmax) {
    if (!trace || D < 1 || !node_stats || !node_dist || !dist || bins < 1 || bins > 64) return fail(B200_ERR_BAD_ARG, "bad argument");
    for (int t = 0; t < D; ++t)
        if (trace[t] < 0 || trace[t] >= M) return fail(B200_ERR_BAD_ARG, "trace index out of range");
    if (b200_device_count() == 0) return fail(B200_ERR_CUDA, "no CUDA device: this library has no CPU path");
    TwinBufs b; float *d_ns = nullptr, *d_nd = nullptr, *d_dist = nullptr;
    TW(b.up(&b.trace, trace, (size_t)D)); TW(b.up(&d_ns, (const float *)node_stats, (size_t)M * 5)); TW(b.up(&d_nd, (const float *)node_dist, (size_t)M * bins));
    TW(b.up(&d_dist, dist, (size_t)bins));
    k_dist_backup_trace<<<1, 32>>>(b.trace, D, d_ns, d_nd, bins, r, d_dist, vmin, vmax);   // the engine's backup (dist_backup_trace_warp)
    CK(cudaGetLastError());
    CK(cudaMemcpy(node_stats, d_ns, (size_t)M * 5 * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(node_dist, d_nd, (size_t)M * bins * 4, cudaMemcpyDeviceToHost));
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- replay samples
__global__ void k_collect_samples(Arena A, int min_visits, uint8_t *out, int capacity, int32_t *count) {
    size_t n = (size_t)A.G * A.M;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        int4 st = A.stat[i];
        if (st.x < min_visits || st.w != 0 || st.x == 0) continue;      // ValueSim.py:143-144 (visit < min or end)
        int slot = atomicAdd(count, 1);
        if (slot >= capacity) continue;
        uint8_t *dst = out + (size_t)slot * 212;
        const uint32_t *k = A.key + i * KEY_WORDS;
        for (int r = 0; r < 20; ++r) {
            uint32_t row = (k[r >> 1] >> ((r & 1) * 16)) & 0x3ffu;
            for (int c = 0; c < 10; ++c) dst[r * 10 + c] = (uint8_t)((row >> c) & 1u);
        }
        for (int j = 0; j < 4; ++j) dst[(k[10] >> (8 * j)) & 0xffu] = 0xff;    // int8 -1
        float f[3] = {__int_as_float(st.y), __int_as_float(st.z), (float)st.x};
        memcpy(dst + 200, f, 12);
    }
}

// Online replay memory (agents/ValueSim.py:14-37, agent.cpp:588-617): allocate `capacity` rows; k_gc appends to it.
extern "C" int b200_replay_enable(b200_engine *e, int min_visits, int capacity) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_enable");
    if (!e || capacity < 1 || min_visits < 0) return fail(B200_ERR_BAD_ARG, "bad argument");
    CK(cudaSetDevice(e->cfg.device));
    if (e->A.replay) return fail(B200_ERR_BAD_ARG, "replay memory already enabled");
    // twice the capacity is allocated: accumulation policy 0 (b200_replay_policy) stages the rows of a collection past memory_size before its
    // random drop decides which of them stay (agent.cpp:800-801); k_gc itself never stores past A.replay_cap
    if (dalloc(e, &e->A.replay, (size_t)2 * capacity * 212) || dalloc(e, &e->A.replay_count, 1)) return B200_ERR_CUDA;
    e->replay_alloc = 2 * capacity;
    e->A.replay_cap = capacity; e->A.replay_min_visits = min_visits;
    e->rp.memory_size = capacity;
    drop_step_graph(e);
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// Hand the stored rows to the trainer / the all-gather: copies min(count, capacity) rows to out_dev (DEVICE) and empties the memory
// (memory_index = 0 after training, ValueSim.py:183 / agent.cpp:700).
extern "C" int b200_replay_drain_dev(b200_engine *e, void *out_dev, int capacity, int32_t *count_out) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_drain_dev");
    if (!e || !out_dev || !count_out || !e->A.replay) return fail(B200_ERR_BAD_ARG, "replay memory not enabled / bad argument");
    CK(cudaSetDevice(e->cfg.device));
    int32_t n = 0;
    CK(cudaMemcpyAsync(&n, e->A.replay_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (n > e->A.replay_cap) n = e->A.replay_cap;
    if (n > capacity) n = capacity;
    if (n > 0) CK(cudaMemcpyAsync(out_dev, e->A.replay, (size_t)n * 212, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemsetAsync(e->A.replay_count, 0, 4, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    *count_out = n;
    return B200_OK;
}

extern "C" int b200_collect_samples_dev(b200_engine *e, int min_visits, void *out_dev, int capacity, int32_t *count_out) {
    if (!e || !out_dev || capacity < 0 || !count_out) return fail(B200_ERR_BAD_ARG, "bad argument");
    CK(cudaSetDevice(e->cfg.device));
    if (!e->d_sample_count) { if (dalloc(e, &e->d_sample_count, 1)) return B200_ERR_CUDA; }
    CK(cudaMemsetAsync(e->d_sample_count, 0, 4, e->stream));
    k_collect_samples<<<e->n_sm * 4, 256, 0, e->stream>>>(e->A, min_visits, (uint8_t *)out_dev, capacity, e->d_sample_count);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(count_out, e->d_sample_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (*count_out > capacity) *count_out = capacity;
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- replay-memory policies (SURVEY 8f.1)
static int rp_count(b200_engine *e, int32_t *n) {
    CK(cudaMemcpyAsync(n, e->A.replay_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (*n > e->A.replay_cap) *n = e->A.replay_cap;
    return B200_OK;
}
static int rp_set_count(b200_engine *e, int32_t n) {
    CK(cudaMemcpyAsync(e->A.replay_count, &n, 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}
static int rp_scratch(b200_engine *e) {
    if (e->d_rp_tmp) return B200_OK;
    if (dalloc(e, &e->d_rp_tmp, (size_t)e->replay_alloc * 212, false) || dalloc(e, &e->d_rp_keep, (size_t)e->replay_alloc, false) ||
        dalloc(e, &e->d_rp_vis, (size_t)e->replay_alloc, false) || dalloc(e, &e->d_rp_kept, 1)) return B200_ERR_CUDA;
    return B200_OK;
}
// rows [lo, hi) with keep[i] != 0 are packed, in order, at lo, lo+1, ...; everything else in the memory stays as it is (the reference compacts
// in place by copying downwards, so positions past the packed rows keep their old content).  Returns the number of packed rows.
static int rp_compact(b200_engine *e, const std::vector<uint8_t> &keep, int lo, int hi, int *kept) {
    int rc = rp_scratch(e);
    if (rc) return rc;
    CK(cudaMemcpyAsync(e->d_rp_keep, keep.data(), (size_t)hi, cudaMemcpyHostToDevice, e->stream));
    k_replay_compact<<<1, 1024, 0, e->stream>>>(e->A.replay, e->d_rp_keep, lo, hi, e->d_rp_tmp, e->d_rp_kept);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(kept, e->d_rp_kept, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (*kept > 0) CK(cudaMemcpyAsync(e->A.replay + (size_t)lo * 212, e->d_rp_tmp + (size_t)lo * 212, (size_t)*kept * 212, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// OnlineMCTSAgent(accumulation_policy, episodes_per_train, memory_growth_rate) agent.cpp:588-617; memory_size / min_visit = b200_replay_enable's
extern "C" int b200_replay_policy(b200_engine *e, int policy, int episodes_per_train, int memory_growth_rate) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_policy");
    if (!e || !e->A.replay || policy < 0 || policy > 3 || episodes_per_train < 1 || memory_growth_rate < 0) return fail(B200_ERR_BAD_ARG, "replay memory not enabled / bad policy");
    CK(cudaSetDevice(e->cfg.device));
    ReplayPolicy fresh;
    fresh.policy = policy; fresh.memory_size = e->rp.memory_size; fresh.episodes_per_train = episodes_per_train; fresh.memory_growth_rate = memory_growth_rate;
    e->rp = fresh;
    e->A.replay_cap = policy == 0 ? e->replay_alloc : e->rp.memory_size;      // policy 0: rows are staged past memory_size until the drop has decided
    drop_step_graph(e);
    return rp_set_count(e, 0);
}

// weighted_trimming(percentile) agent.cpp:710-749 (literally, including that the first removed row is not subtracted from memory_index)
static int rp_weighted_trimming(b200_engine *e, double percentile) {
    ReplayPolicy &P = e->rp;
    const int N = P.memory_size;
    int rc = rp_scratch(e);
    if (rc) return rc;
    k_replay_visits<<<(N + 255) / 256, 256, 0, e->stream>>>(e->A.replay, N, e->d_rp_vis);
    std::vector<float> vis(N);
    CK(cudaMemcpyAsync(vis.data(), e->d_rp_vis, (size_t)N * 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    std::vector<int> weights(N);
    for (int i = 0; i < N; ++i) weights[i] = (int)vis[i];
    std::sort(weights.begin(), weights.end());
    const int threshold = weights[(int)(N * percentile)];
    int idx_fill = -1;
    for (int i = 0; i < N; ++i) if (vis[i] <= (float)threshold) { idx_fill = i; break; }
    std::vector<uint8_t> keep(N, 1);
    for (int i = idx_fill; i < N; ++i) if (vis[i] <= (float)threshold) keep[i] = 0;
    for (int i = idx_fill + 1; i < N; ++i) if (vis[i] <= (float)threshold) --P.memory_index;
    int kept = 0;
    return rp_compact(e, keep, idx_fill, N, &kept);
}

// random_trimming(fraction) agent.cpp:751-775: IntSampler(memory_size).sample(n) = std::shuffle of the persistent index vector, first n, sorted
static int rp_random_trimming(b200_engine *e, double fraction) {
    ReplayPolicy &P = e->rp;
    const int N = P.memory_size;
    if (P.sampler.empty()) { P.sampler.resize(N); std::iota(P.sampler.begin(), P.sampler.end(), 0); }
    std::shuffle(P.sampler.begin(), P.sampler.end(), P.mt);
    std::vector<int> indices(P.sampler.begin(), P.sampler.begin() + (int)(N * fraction));
    if (indices.empty()) return B200_OK;                          // (the reference reads indices.front() of an empty vector here: UB)
    std::sort(indices.begin(), indices.end());
    std::vector<uint8_t> keep(N, 1);
    for (int i : indices) keep[i] = 0;
    P.memory_index -= (int)indices.size();
    int kept = 0;
    return rp_compact(e, keep, indices.front(), N, &kept);
}

// The policy half of OnlineMCTSAgent::remove_nodes (agent.cpp:632-702), to be called after the collection(s) that stored rows — the reference
// runs it inside every remove_nodes(); a single-game engine calls it after every simulation step / update_root in which counter 3 (collections)
// moved and then reproduces the reference exactly; a batched run calls it once per move.  current_episode = Agent::current_episode
// (agent.cpp:69,279-280: games finished so far).  *train_now = the reference would call train(m_state, m_value, m_variance, m_visit, memory_index)
// now: drain the first *memory_index rows (b200_replay_peek_dev), train, then b200_replay_policy_trained().
extern "C" int b200_replay_policy_step(b200_engine *e, int64_t current_episode, int32_t *train_now, int32_t *memory_index) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_policy_step");
    if (!e || !train_now || !memory_index || e->rp.policy < 0) return fail(B200_ERR_BAD_ARG, "no replay policy configured");
    CK(cudaSetDevice(e->cfg.device));
    ReplayPolicy &P = e->rp;
    int32_t count = 0;
    int rc = rp_count(e, &count);
    if (rc) return rc;
    const int cur = (int)current_episode;
    if (P.policy == 0) {
        // store_nodes' drop (agent.cpp:798-801), applied to the rows this collection staged, in their order: ++accumulated_nodes; a row is dropped
        // with probability memory_drop_prob; storing stops when the memory is full (:817)
        std::vector<uint8_t> keep((size_t)std::max(count, 1), 1);
        int kept_total = P.memory_index;
        bool full = kept_total >= P.memory_size;
        for (int i = P.memory_index; i < count; ++i) {
            if (full) { keep[i] = 0; continue; }
            ++P.accumulated_nodes;
            if (P.unif(P.mt) < P.memory_drop_prob) { keep[i] = 0; continue; }
            if (++kept_total == P.memory_size) full = true;
        }
        if (count > P.memory_index) {
            int kept = 0;
            rc = rp_compact(e, keep, P.memory_index, count, &kept);
            if (rc) return rc;
        }
        P.memory_index = kept_total;
        rc = rp_set_count(e, P.memory_index);
        if (rc) return rc;
    } else {
        P.memory_index = count < P.memory_size ? count : P.memory_size;
    }
    bool pass = false;
    const int diff = cur - P.last_training_episode;
    if (P.policy == 0) {
        if (P.last_accumulation_episode != cur) {
            P.nodes_per_episode.push_back(P.accumulated_nodes);
            if ((int)P.nodes_per_episode.size() > P.episodes_per_train) P.nodes_per_episode.pop_front();
            const int sum = std::accumulate(P.nodes_per_episode.begin(), P.nodes_per_episode.end(), 0);
            P.memory_drop_prob = std::max(0., 1. - double(P.memory_size) / sum);
            P.accumulated_nodes = 0;
            P.last_accumulation_episode = cur;
        }
        pass = diff >= P.episodes_per_train;
        if (!pass && P.memory_index >= P.memory_size) { rc = rp_random_trimming(e, 0.01); if (rc) return rc; rc = rp_set_count(e, P.memory_index); if (rc) return rc; }
    } else if (P.policy == 1) {
        pass = diff >= P.episodes_per_train;
        if (!pass && P.memory_index >= P.memory_size) { rc = rp_weighted_trimming(e, 0.01); if (rc) return rc; rc = rp_set_count(e, P.memory_index); if (rc) return rc; }
    } else if (P.policy == 2) {
        pass = diff >= P.episodes_per_train || P.memory_index >= P.memory_size;
    } else {
        const int m_size = std::min(P.n_trains * P.memory_growth_rate, P.memory_size);
        pass = P.memory_index >= m_size;
    }
    *train_now = pass ? 1 : 0;
    *memory_index = P.memory_index;
    return B200_OK;
}

// after train(...): ++n_trains; memory_index = 0; last_training_episode = current_episode (agent.cpp:697-701)
extern "C" int b200_replay_policy_trained(b200_engine *e, int64_t current_episode) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_policy_trained");
    if (!e || e->rp.policy < 0) return fail(B200_ERR_BAD_ARG, "no replay policy configured");
    CK(cudaSetDevice(e->cfg.device));
    e->rp.n_trains += 1;
    e->rp.memory_index = 0;
    e->rp.last_training_episode = (int)current_episode;
    return rp_set_count(e, 0);
}

// Append n rows (HOST, 212 bytes each, the format k_gc stores) to the memory exactly as a collection would: in order, until the memory is full
// (agent.cpp:817).  Seeds the memory from a dump file (ValueSim.py:176-177) or from another process; the policy tests script collections with it.
extern "C" int b200_replay_append(b200_engine *e, const uint8_t *rows, int n) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_append");
    if (!e || !e->A.replay || (n > 0 && !rows) || n < 0) return fail(B200_ERR_BAD_ARG, "replay memory not enabled / bad argument");
    CK(cudaSetDevice(e->cfg.device));
    int32_t count = 0;
    int rc = rp_count(e, &count);
    if (rc) return rc;
    int take = e->A.replay_cap - count;
    if (take > n) take = n;
    if (take > 0) CK(cudaMemcpyAsync(e->A.replay + (size_t)count * 212, rows, (size_t)take * 212, cudaMemcpyHostToDevice, e->stream));
    return rp_set_count(e, count + (take > 0 ? take : 0));
}

// b200_replay_append from a DEVICE buffer: rank 0 of a data-parallel run appends the rows the other ranks' collections stored this move
extern "C" int b200_replay_append_dev(b200_engine *e, const void *rows, int n) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_append_dev");
    if (!e || !e->A.replay || (n > 0 && !rows) || n < 0) return fail(B200_ERR_BAD_ARG, "replay memory not enabled / bad argument");
    CK(cudaSetDevice(e->cfg.device));
    int32_t count = 0;
    int rc = rp_count(e, &count);
    if (rc) return rc;
    int take = e->A.replay_cap - count;
    if (take > n) take = n;
    if (take > 0) CK(cudaMemcpyAsync(e->A.replay + (size_t)count * 212, rows, (size_t)take * 212, cudaMemcpyDeviceToDevice, e->stream));
    return rp_set_count(e, count + (take > 0 ? take : 0));
}

// the first n rows of the memory, copied to a DEVICE buffer without emptying it (the arrays the reference hands to train(): m_state ... [:memory_index])
extern "C" int b200_replay_peek_dev(b200_engine *e, void *out_dev, int n) {
    if (e) REFUSE_IF_OPEN(e, "b200_replay_peek_dev");
    if (!e || !out_dev || n < 0 || !e->A.replay || n > e->replay_alloc) return fail(B200_ERR_BAD_ARG, "bad argument");
    CK(cudaSetDevice(e->cfg.device));
    if (n > 0) CK(cudaMemcpyAsync(out_dev, e->A.replay, (size_t)n * 212, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- snapshot (b200_engine_save / _load)
// File: "B200SNAP", u32 version, u32 byte-order mark, then fields {u32 id, u32 0, u64 nbytes, payload, u64 checksum(payload)}; the arena field
// comes last but one and carries its own layout (u64 n_games, u64 words[n_games], u64 checksum(words), the packed games of snapshot.cuh,
// each with its device checksum); a field of id 0 ends the file.  Scalars are 8-byte payloads (int64, or the bits of a double).
namespace {

constexpr char SNAP_MAGIC[8] = {'B', '2', '0', '0', 'S', 'N', 'A', 'P'};
constexpr uint32_t SNAP_VERSION = 1, SNAP_BOM = 0x01020304u;
enum : uint32_t {
    F_END = 0,
    // b200_config, one field each
    F_N_GAMES = 1, F_MAX_NODES, F_MODE, F_LOW, F_LP_END_FROM_OBS, F_LP_VAR_GAMMA2, F_STALE_POP, F_OVERFLOW_RESET, F_EVAL_KIND, F_TRACE_MAX,
    F_ACTIONS_PER_DROP, F_SCORING, F_RANDOMIZER, F_DEVICE, F_SEED, F_GAMMA, F_ROLLOUT_VARIANCE, F_DIST_BINS, F_DIST_VMIN, F_DIST_VMAX,
    // engine settings that change results or run shape
    F_PATH_CACHE = 32, F_DEEP_CAP, F_GC_HEADROOM,
    // networks, as b200_load_weights / b200_load_dist_weights took them
    F_WEIGHTS = 40, F_DIST_ATOMS, F_DIST_WEIGHTS,
    F_COUNTERS = 48, F_FIN_COUNT, F_FIN_LOG,
    // replay memory and its policy (ReplayPolicy)
    F_REPLAY_MIN_VISITS = 56, F_REPLAY_CAPACITY, F_REPLAY_CAP, F_REPLAY_COUNT, F_REPLAY_ROWS,
    F_RP_POLICY = 64, F_RP_MEMORY_SIZE, F_RP_EPISODES_PER_TRAIN, F_RP_GROWTH, F_RP_MEMORY_INDEX, F_RP_ACCUMULATED, F_RP_LAST_ACCUMULATION,
    F_RP_LAST_TRAINING, F_RP_N_TRAINS, F_RP_DROP_PROB, F_RP_NODES_PER_EPISODE, F_RP_MT, F_RP_SAMPLER,
    F_ARENA = 128,
};
static bool snap_known(uint32_t id) {
    return (id >= F_N_GAMES && id <= F_DIST_VMAX) || (id >= F_PATH_CACHE && id <= F_GC_HEADROOM) || (id >= F_WEIGHTS && id <= F_DIST_WEIGHTS) ||
           (id >= F_COUNTERS && id <= F_FIN_LOG) || (id >= F_REPLAY_MIN_VISITS && id <= F_REPLAY_ROWS) || (id >= F_RP_POLICY && id <= F_RP_SAMPLER);
}

int64_t g_snap_staging = 64ll << 20;   // b200_snapshot_set_staging
thread_local double g_snap_sec[6];      // pack, D2H, write | read, H2D, unpack of this thread's last save | load

uint64_t host_checksum(const void *p, size_t n, uint64_t h = 0xcbf29ce484222325ull) {   // FNV-1a over 8-byte words, then the tail bytes
    const uint8_t *b = (const uint8_t *)p;
    size_t i = 0;
    for (; i + 8 <= n; i += 8) { uint64_t w; memcpy(&w, b + i, 8); h = (h ^ w) * 0x100000001b3ull; }
    for (; i < n; ++i) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}
double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Pinned {   // the two host halves of the staging buffer
    void *p = nullptr;
    ~Pinned() { if (p) cudaFreeHost(p); }
};
struct Events {
    std::vector<cudaEvent_t> ev;
    ~Events() { for (auto x : ev) cudaEventDestroy(x); }
    cudaEvent_t make() { cudaEvent_t x = nullptr; cudaEventCreate(&x); ev.push_back(x); return x; }
};

struct Writer {
    FILE *f = nullptr;
    bool ok = true;
    void raw(const void *p, size_t n) { if (ok && n && fwrite(p, 1, n, f) != n) ok = false; }
    void field(uint32_t id, const void *p, uint64_t n) {
        const uint32_t hdr[2] = {id, 0u};
        raw(hdr, 8); raw(&n, 8); raw(p, n);
        const uint64_t cs = host_checksum(p, n);
        raw(&cs, 8);
    }
    void i64(uint32_t id, int64_t v) { field(id, &v, 8); }
    void f64(uint32_t id, double v) { field(id, &v, 8); }
};

struct Reader {
    FILE *f = nullptr;
    uint64_t left = 0;                   // bytes of the file not read yet
    bool raw(void *p, uint64_t n) { if (n > left || fread(p, 1, n, f) != n) return false; left -= n; return true; }
};

// the staging halves: each holds the largest game; chunks of whole games of at most `half` bytes
static size_t snap_half(const std::vector<long long> &words) {
    long long most = 0;
    for (long long w : words) most = std::max(most, w);
    return std::max<size_t>((size_t)(g_snap_staging / 2), (size_t)most * 4);
}

}  // namespace

extern "C" int b200_snapshot_set_staging(int64_t bytes) {
    g_snap_staging = bytes > 0 ? bytes : (64ll << 20);
    return B200_OK;
}

extern "C" int b200_snapshot_timing(double *sec6) {
    if (!sec6) return fail(B200_ERR_BAD_ARG, "null argument");
    memcpy(sec6, g_snap_sec, sizeof(g_snap_sec));
    return B200_OK;
}

extern "C" int b200_engine_save(b200_engine *e, const char *path, int64_t *bytes_out) {
    if (!e || !path) return fail(B200_ERR_BAD_ARG, "null argument");
    REFUSE_IF_OPEN(e, "b200_engine_save");
    CK(cudaSetDevice(e->cfg.device));
    CK(cudaStreamSynchronize(e->stream));
    if (e->stream1) CK(cudaStreamSynchronize(e->stream1));
    for (double &s : g_snap_sec) s = 0.0;
    const Arena &A = e->A;
    const int G = A.G;
    // sizes of the packed games
    Scratch tmp;
    long long *d_words = nullptr, *d_off = nullptr; int32_t *d_ent = nullptr;
    CK(tmp.get(&d_words, (size_t)G * 8)); CK(tmp.get(&d_ent, (size_t)G * 8)); CK(tmp.get(&d_off, (size_t)(G + 1) * 8));
    k_snap_count<<<G, 256, 0, e->stream>>>(A, d_words, d_ent);
    CK(cudaGetLastError());
    std::vector<long long> words(G), off(G + 1, 0);
    CK(cudaMemcpyAsync(words.data(), d_words, (size_t)G * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    for (int g = 0; g < G; ++g) off[g + 1] = off[g] + words[g];
    CK(cudaMemcpyAsync(d_off, off.data(), (size_t)(G + 1) * 8, cudaMemcpyHostToDevice, e->stream));
    // the host-side state
    std::vector<uint64_t> counters(48);
    int32_t fin_count = 0, replay_count = 0;
    CK(cudaMemcpyAsync(counters.data(), A.counters, 48 * 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaMemcpyAsync(&fin_count, A.fin_count, 4, cudaMemcpyDeviceToHost, e->stream));
    if (A.replay) CK(cudaMemcpyAsync(&replay_count, A.replay_count, 4, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    std::vector<int32_t> fin((size_t)std::min(fin_count, A.fin_cap) * 4);
    if (!fin.empty()) CK(cudaMemcpy(fin.data(), A.fin_log, fin.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<uint8_t> rows;
    if (A.replay) {
        rows.resize((size_t)std::max(0, std::min(replay_count, e->replay_alloc)) * 212);
        if (!rows.empty()) CK(cudaMemcpy(rows.data(), A.replay, rows.size(), cudaMemcpyDeviceToHost));
    }
    // staging: two device halves and two pinned halves, packed / copied / written in turn
    const size_t half = snap_half(words);
    uint8_t *d_stage = nullptr;
    CK(tmp.get(&d_stage, 2 * half));
    Pinned pin;
    CK(cudaHostAlloc(&pin.p, 2 * half, cudaHostAllocDefault));
    const std::string tmp_path = std::string(path) + ".tmp";
    Writer W;
    W.f = fopen(tmp_path.c_str(), "wb");
    if (!W.f) return fail(B200_ERR_BAD_ARG, "b200_engine_save: cannot open " + tmp_path + " for writing: " + strerror(errno));
    struct Closer { Writer &w; std::string p; bool keep = false; ~Closer() { if (w.f) fclose(w.f); if (!keep) remove(p.c_str()); } } closer{W, tmp_path};
    W.raw(SNAP_MAGIC, 8); W.raw(&SNAP_VERSION, 4); W.raw(&SNAP_BOM, 4);
    const b200_config &c = e->cfg;
    W.i64(F_N_GAMES, c.n_games); W.i64(F_MAX_NODES, c.max_nodes); W.i64(F_MODE, c.mode); W.i64(F_LOW, c.low);
    W.i64(F_LP_END_FROM_OBS, c.lp_end_from_obs); W.i64(F_LP_VAR_GAMMA2, c.lp_var_gamma2); W.i64(F_STALE_POP, c.stale_pop);
    W.i64(F_OVERFLOW_RESET, c.overflow_reset); W.i64(F_EVAL_KIND, c.eval_kind); W.i64(F_TRACE_MAX, c.trace_max);
    W.i64(F_ACTIONS_PER_DROP, c.actions_per_drop); W.i64(F_SCORING, c.scoring); W.i64(F_RANDOMIZER, c.randomizer); W.i64(F_DEVICE, c.device);
    W.i64(F_SEED, c.seed); W.f64(F_GAMMA, c.gamma); W.f64(F_ROLLOUT_VARIANCE, c.rollout_variance); W.i64(F_DIST_BINS, c.dist_bins);
    W.f64(F_DIST_VMIN, c.dist_vmin); W.f64(F_DIST_VMAX, c.dist_vmax);
    W.i64(F_PATH_CACHE, A.pc != nullptr); W.i64(F_DEEP_CAP, e->deep_cap); W.i64(F_GC_HEADROOM, e->gc_headroom);
    if (e->have_weights) W.field(F_WEIGHTS, e->h_w.data(), e->h_w.size() * 4);
    if (e->have_dist_weights) { W.i64(F_DIST_ATOMS, e->dn_atoms); W.field(F_DIST_WEIGHTS, e->h_dnw.data(), e->h_dnw.size() * 4); }
    W.field(F_COUNTERS, counters.data(), counters.size() * 8);
    W.i64(F_FIN_COUNT, fin_count);
    W.field(F_FIN_LOG, fin.data(), fin.size() * 4);
    if (A.replay) {
        W.i64(F_REPLAY_MIN_VISITS, A.replay_min_visits); W.i64(F_REPLAY_CAPACITY, e->replay_alloc / 2); W.i64(F_REPLAY_CAP, A.replay_cap);
        W.i64(F_REPLAY_COUNT, replay_count); W.field(F_REPLAY_ROWS, rows.data(), rows.size());
    }
    if (e->rp.policy >= 0) {
        const ReplayPolicy &P = e->rp;
        W.i64(F_RP_POLICY, P.policy); W.i64(F_RP_MEMORY_SIZE, P.memory_size); W.i64(F_RP_EPISODES_PER_TRAIN, P.episodes_per_train);
        W.i64(F_RP_GROWTH, P.memory_growth_rate); W.i64(F_RP_MEMORY_INDEX, P.memory_index); W.i64(F_RP_ACCUMULATED, P.accumulated_nodes);
        W.i64(F_RP_LAST_ACCUMULATION, P.last_accumulation_episode); W.i64(F_RP_LAST_TRAINING, P.last_training_episode);
        W.i64(F_RP_N_TRAINS, P.n_trains); W.f64(F_RP_DROP_PROB, P.memory_drop_prob);
        const std::vector<int32_t> npe(P.nodes_per_episode.begin(), P.nodes_per_episode.end());
        W.field(F_RP_NODES_PER_EPISODE, npe.data(), npe.size() * 4);
        std::ostringstream mt;
        mt << P.mt;
        const std::string s = mt.str();
        W.field(F_RP_MT, s.data(), s.size());
        W.field(F_RP_SAMPLER, P.sampler.data(), P.sampler.size() * 4);
    }
    // the arena
    {
        const uint32_t hdr[2] = {F_ARENA, 0u};
        const uint64_t G64 = (uint64_t)G, nbytes = 8 + 8 * G64 + 8 + (uint64_t)off[G] * 4;
        std::vector<uint64_t> w64(words.begin(), words.end());
        const uint64_t cs = host_checksum(w64.data(), w64.size() * 8);
        W.raw(hdr, 8); W.raw(&nbytes, 8); W.raw(&G64, 8); W.raw(w64.data(), w64.size() * 8); W.raw(&cs, 8);
    }
    Events ev;
    const int grid_max = e->gc_pool_main;
    std::vector<std::array<cudaEvent_t, 3>> chunk_ev;
    std::vector<std::pair<size_t, int>> pending;   // (bytes, buffer) of the chunk copied but not written yet
    auto write_chunk = [&](size_t bytes, int buf, cudaEvent_t done) -> int {
        CK(cudaEventSynchronize(done));
        const double t0 = now_s();
        W.raw((uint8_t *)pin.p + buf * half, bytes);
        g_snap_sec[2] += now_s() - t0;
        return B200_OK;
    };
    int g0 = 0, k = 0;
    size_t prev_bytes = 0; int prev_buf = -1; cudaEvent_t prev_done = nullptr;
    while (g0 < G) {
        int g1 = g0;
        while (g1 < G && (size_t)(off[g1 + 1] - off[g0]) * 4 <= half) ++g1;
        const int buf = k & 1;
        const size_t bytes = (size_t)(off[g1] - off[g0]) * 4;
        std::array<cudaEvent_t, 3> ce{ev.make(), ev.make(), ev.make()};
        CK(cudaEventRecord(ce[0], e->stream));
        k_snap_pack<<<std::min(grid_max, g1 - g0), GC_THREADS, 0, e->stream>>>(A, g0, g1, d_off, off[g0], d_ent, (uint32_t *)(d_stage + buf * half));
        CK(cudaGetLastError());
        CK(cudaEventRecord(ce[1], e->stream));
        // the pinned half this chunk lands in was written out two chunks ago (write_chunk below runs in order)
        CK(cudaMemcpyAsync((uint8_t *)pin.p + buf * half, d_stage + buf * half, bytes, cudaMemcpyDeviceToHost, e->stream));
        CK(cudaEventRecord(ce[2], e->stream));
        chunk_ev.push_back(ce);
        if (prev_buf >= 0) { int rc = write_chunk(prev_bytes, prev_buf, prev_done); if (rc) return rc; }
        prev_bytes = bytes; prev_buf = buf; prev_done = ce[2];
        g0 = g1; ++k;
    }
    if (prev_buf >= 0) { int rc = write_chunk(prev_bytes, prev_buf, prev_done); if (rc) return rc; }
    CK(cudaStreamSynchronize(e->stream));
    for (auto &ce : chunk_ev) {
        float a = 0.f, b = 0.f;
        cudaEventElapsedTime(&a, ce[0], ce[1]); cudaEventElapsedTime(&b, ce[1], ce[2]);
        g_snap_sec[0] += a * 1e-3; g_snap_sec[1] += b * 1e-3;
    }
    {
        const uint32_t end[2] = {F_END, 0u};
        const uint64_t zero = 0;
        W.raw(end, 8); W.raw(&zero, 8); W.raw(&zero, 8);
    }
    const double t0 = now_s();
    if (W.ok && fflush(W.f) != 0) W.ok = false;
    if (W.ok && fsync(fileno(W.f)) != 0) W.ok = false;
    const long long total = W.ok ? (long long)ftello(W.f) : -1;
    g_snap_sec[2] += now_s() - t0;
    if (!W.ok) return fail(B200_ERR_BAD_ARG, "b200_engine_save: writing " + tmp_path + " failed: " + strerror(errno));
    fclose(W.f); W.f = nullptr;
    if (rename(tmp_path.c_str(), path) != 0) return fail(B200_ERR_BAD_ARG, std::string("b200_engine_save: rename to ") + path + " failed: " + strerror(errno));
    closer.keep = true;
    if (bytes_out) *bytes_out = total;
    return B200_OK;
}

namespace {
struct Fields {
    std::map<uint32_t, std::vector<uint8_t>> v;
    bool has(uint32_t id) const { return v.count(id) != 0; }
    bool scalar(uint32_t id, int64_t &out) const {
        auto it = v.find(id);
        if (it == v.end() || it->second.size() != 8) return false;
        memcpy(&out, it->second.data(), 8);
        return true;
    }
    bool real(uint32_t id, double &out) const {
        auto it = v.find(id);
        if (it == v.end() || it->second.size() != 8) return false;
        memcpy(&out, it->second.data(), 8);
        return true;
    }
};
}  // namespace

static int snap_bad(const std::string &path, const std::string &why) { return fail(B200_ERR_BAD_ARG, "b200_engine_load: " + path + ": " + why); }

// everything of the engine but its arena, from the fields before it
static int snap_restore_host(b200_engine *e, const Fields &F, const std::string &path) {
    int64_t v = 0;
    int rc = 0;
    if (F.scalar(F_GC_HEADROOM, v)) e->gc_headroom = (int)v;
    if (F.scalar(F_PATH_CACHE, v) && v) { rc = b200_set_path_cache(e, 1); if (rc) return rc; }   // saved on, restored with an empty cache
    if (F.scalar(F_DEEP_CAP, v) && v) { rc = b200_set_deep_lane(e, (int)v); if (rc) return rc; }
    if (F.has(F_WEIGHTS)) {
        const auto &w = F.v.at(F_WEIGHTS);
        if (w.size() != (size_t)B200_N_WEIGHTS * 4) return snap_bad(path, "value weights of the wrong size");
        rc = b200_load_weights(e, reinterpret_cast<const float *>(w.data()));
        if (rc) return rc;
    }
    if (F.has(F_DIST_WEIGHTS)) {
        int64_t atoms = 0;
        if (!F.scalar(F_DIST_ATOMS, atoms) || atoms < 2 || atoms > 64 || F.v.at(F_DIST_WEIGHTS).size() != dn_weight_count((int)atoms) * 4)
            return snap_bad(path, "distributional weights of the wrong size");
        rc = b200_load_dist_weights(e, reinterpret_cast<const float *>(F.v.at(F_DIST_WEIGHTS).data()), (int)atoms);
        if (rc) return rc;
    }
    Arena &A = e->A;
    const auto &cnt = F.v.count(F_COUNTERS) ? F.v.at(F_COUNTERS) : std::vector<uint8_t>();
    if (cnt.size() != 48 * 8) return snap_bad(path, "counters missing");
    int64_t fin_count = 0;
    if (!F.scalar(F_FIN_COUNT, fin_count) || fin_count < 0 || !F.has(F_FIN_LOG) ||
        F.v.at(F_FIN_LOG).size() != (size_t)std::min<int64_t>(fin_count, A.fin_cap) * 16)
        return snap_bad(path, "finished-games log inconsistent");
    CK(cudaMemcpyAsync(A.counters, cnt.data(), cnt.size(), cudaMemcpyHostToDevice, e->stream));
    const int32_t fc = (int32_t)fin_count;
    CK(cudaMemcpyAsync(A.fin_count, &fc, 4, cudaMemcpyHostToDevice, e->stream));
    if (!F.v.at(F_FIN_LOG).empty()) CK(cudaMemcpyAsync(A.fin_log, F.v.at(F_FIN_LOG).data(), F.v.at(F_FIN_LOG).size(), cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (F.has(F_REPLAY_CAPACITY)) {
        int64_t mv = 0, cap = 0, rcap = 0, count = 0;
        if (!F.scalar(F_REPLAY_MIN_VISITS, mv) || !F.scalar(F_REPLAY_CAPACITY, cap) || !F.scalar(F_REPLAY_CAP, rcap) || !F.scalar(F_REPLAY_COUNT, count) ||
            !F.has(F_REPLAY_ROWS) || cap < 1 || cap > (1 << 29) || rcap < 0 || rcap > 2 * cap || count < 0 ||
            F.v.at(F_REPLAY_ROWS).size() != (size_t)std::min<int64_t>(count, 2 * cap) * 212)
            return snap_bad(path, "replay memory fields inconsistent");
        rc = b200_replay_enable(e, (int)mv, (int)cap);
        if (rc) return rc;
        const auto &rows = F.v.at(F_REPLAY_ROWS);
        if (!rows.empty()) CK(cudaMemcpyAsync(A.replay, rows.data(), rows.size(), cudaMemcpyHostToDevice, e->stream));
        A.replay_cap = (int)rcap;
        rc = rp_set_count(e, (int32_t)count);
        if (rc) return rc;
    }
    if (F.has(F_RP_POLICY)) {
        if (!A.replay) return snap_bad(path, "a replay policy without a replay memory");
        ReplayPolicy P;
        int64_t x[9];
        const uint32_t ids[9] = {F_RP_POLICY, F_RP_MEMORY_SIZE, F_RP_EPISODES_PER_TRAIN, F_RP_GROWTH, F_RP_MEMORY_INDEX, F_RP_ACCUMULATED,
                                 F_RP_LAST_ACCUMULATION, F_RP_LAST_TRAINING, F_RP_N_TRAINS};
        for (int i = 0; i < 9; ++i) if (!F.scalar(ids[i], x[i])) return snap_bad(path, "replay policy field " + std::to_string(ids[i]) + " missing");
        if (x[0] < 0 || x[0] > 3 || x[1] != e->replay_alloc / 2) return snap_bad(path, "replay policy inconsistent with the memory");
        P.policy = (int)x[0]; P.memory_size = (int)x[1]; P.episodes_per_train = (int)x[2]; P.memory_growth_rate = (int)x[3]; P.memory_index = (int)x[4];
        P.accumulated_nodes = (int)x[5]; P.last_accumulation_episode = (int)x[6]; P.last_training_episode = (int)x[7]; P.n_trains = (int)x[8];
        if (!F.real(F_RP_DROP_PROB, P.memory_drop_prob) || !F.has(F_RP_NODES_PER_EPISODE) || !F.has(F_RP_MT) || !F.has(F_RP_SAMPLER))
            return snap_bad(path, "replay policy fields missing");
        const auto &npe = F.v.at(F_RP_NODES_PER_EPISODE), &smp = F.v.at(F_RP_SAMPLER), &mt = F.v.at(F_RP_MT);
        if (npe.size() % 4 || smp.size() % 4 || (!smp.empty() && smp.size() != (size_t)P.memory_size * 4)) return snap_bad(path, "replay policy lists malformed");
        for (size_t i = 0; i < npe.size(); i += 4) { int32_t q; memcpy(&q, &npe[i], 4); P.nodes_per_episode.push_back(q); }
        P.sampler.resize(smp.size() / 4);
        if (!smp.empty()) memcpy(P.sampler.data(), smp.data(), smp.size());
        for (int s : P.sampler) if (s < 0 || s >= P.memory_size) return snap_bad(path, "replay policy sampler index out of range");
        std::istringstream in(std::string(mt.begin(), mt.end()));
        in >> P.mt;
        if (in.fail()) return snap_bad(path, "replay policy random state malformed");
        e->rp = P;
    }
    return B200_OK;
}

extern "C" int b200_engine_load(const char *path, int device, b200_engine **out) {
    if (!path || !out) return fail(B200_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    for (double &s : g_snap_sec) s = 0.0;
    const std::string P = path;
    Reader R;
    R.f = fopen(path, "rb");
    if (!R.f) return snap_bad(P, std::string("cannot open: ") + strerror(errno));
    struct FileGuard { FILE *f; ~FileGuard() { fclose(f); } } fguard{R.f};
    if (fseeko(R.f, 0, SEEK_END) != 0) return snap_bad(P, "not seekable");
    R.left = (uint64_t)ftello(R.f);
    fseeko(R.f, 0, SEEK_SET);
    char magic[8]; uint32_t version = 0, bom = 0;
    if (!R.raw(magic, 8) || !R.raw(&version, 4) || !R.raw(&bom, 4)) return snap_bad(P, "truncated header");
    if (memcmp(magic, SNAP_MAGIC, 8) != 0) return snap_bad(P, "not an engine image (wrong magic)");
    if (bom != SNAP_BOM) return snap_bad(P, "written with another byte order");
    if (version != SNAP_VERSION) return snap_bad(P, "format version " + std::to_string(version) + ", this library reads version " + std::to_string(SNAP_VERSION));
    Fields F;
    uint32_t hdr[2]; uint64_t nbytes = 0;
    for (;;) {
        if (!R.raw(hdr, 8) || !R.raw(&nbytes, 8)) return snap_bad(P, "truncated");
        if (hdr[0] == F_ARENA) break;
        if (hdr[0] == F_END) return snap_bad(P, "no arena");
        if (!snap_known(hdr[0]) || hdr[1] != 0u) return snap_bad(P, "unknown field " + std::to_string(hdr[0]));
        if (F.has(hdr[0])) return snap_bad(P, "field " + std::to_string(hdr[0]) + " twice");
        if (nbytes > R.left || R.left - nbytes < 8) return snap_bad(P, "truncated");
        std::vector<uint8_t> b(nbytes);
        uint64_t cs = 0;
        if (!R.raw(b.data(), nbytes) || !R.raw(&cs, 8)) return snap_bad(P, "truncated");
        if (cs != host_checksum(b.data(), b.size())) return snap_bad(P, "field " + std::to_string(hdr[0]) + ": checksum mismatch");
        F.v[hdr[0]] = std::move(b);
    }
    // the configuration: every field present
    b200_config c;
    memset(&c, 0, sizeof(c));
    {
        int64_t x[15];
        const uint32_t ids[15] = {F_N_GAMES, F_MAX_NODES, F_MODE, F_LOW, F_LP_END_FROM_OBS, F_LP_VAR_GAMMA2, F_STALE_POP, F_OVERFLOW_RESET,
                                  F_EVAL_KIND, F_TRACE_MAX, F_ACTIONS_PER_DROP, F_SCORING, F_RANDOMIZER, F_DEVICE, F_SEED};
        for (int i = 0; i < 15; ++i) if (!F.scalar(ids[i], x[i])) return snap_bad(P, "configuration field " + std::to_string(ids[i]) + " missing");
        int64_t bins = 0;
        if (!F.real(F_GAMMA, c.gamma) || !F.real(F_ROLLOUT_VARIANCE, c.rollout_variance) || !F.scalar(F_DIST_BINS, bins) ||
            !F.real(F_DIST_VMIN, c.dist_vmin) || !F.real(F_DIST_VMAX, c.dist_vmax))
            return snap_bad(P, "configuration incomplete");
        c.n_games = (int32_t)x[0]; c.max_nodes = (int32_t)x[1]; c.mode = (int32_t)x[2]; c.low = (int32_t)x[3]; c.lp_end_from_obs = (int32_t)x[4];
        c.lp_var_gamma2 = (int32_t)x[5]; c.stale_pop = (int32_t)x[6]; c.overflow_reset = (int32_t)x[7]; c.eval_kind = (int32_t)x[8];
        c.trace_max = (int32_t)x[9]; c.actions_per_drop = (int32_t)x[10]; c.scoring = (int32_t)x[11]; c.randomizer = (int32_t)x[12];
        c.device = device >= 0 ? device : (int32_t)x[13]; c.seed = (uint32_t)x[14]; c.dist_bins = (int32_t)bins;
        if (x[0] < 1 || x[0] > (1 << 24)) return snap_bad(P, "n_games out of range");
    }
    // the arena's framing, checked before anything is allocated
    const int G = c.n_games;
    uint64_t G64 = 0;
    if (!R.raw(&G64, 8) || G64 != (uint64_t)G) return snap_bad(P, "arena of another number of games");
    std::vector<uint64_t> w64(G);
    uint64_t wcs = 0;
    if (!R.raw(w64.data(), (uint64_t)G * 8) || !R.raw(&wcs, 8)) return snap_bad(P, "truncated");
    if (wcs != host_checksum(w64.data(), w64.size() * 8)) return snap_bad(P, "arena size table: checksum mismatch");
    std::vector<long long> words(G), off(G + 1, 0);
    for (int g = 0; g < G; ++g) {
        if (w64[g] < (uint64_t)SNAP_HDR + 2 || w64[g] > (1ull << 40)) return snap_bad(P, "game " + std::to_string(g) + ": size out of range");
        words[g] = (long long)w64[g];
        off[g + 1] = off[g] + words[g];
    }
    if (nbytes != 8 + 8 * (uint64_t)G + 8 + (uint64_t)off[G] * 4) return snap_bad(P, "arena length does not match its games");
    if ((uint64_t)off[G] * 4 + 24 > R.left) return snap_bad(P, "truncated");
    // the engine
    b200_engine *e = nullptr;
    int rc = b200_engine_create(&c, &e);
    if (rc) return rc;
    struct Guard { b200_engine *e; ~Guard() { if (e) b200_engine_destroy(e); } } guard{e};
    rc = snap_restore_host(e, F, P);
    if (rc) return rc;
    F.v.clear();
    const Arena &A = e->A;
    const size_t half = snap_half(words);
    Scratch tmp;
    uint8_t *d_stage = nullptr; long long *d_off = nullptr; unsigned long long *d_err = nullptr;
    CK(tmp.get(&d_stage, 2 * half)); CK(tmp.get(&d_off, (size_t)(G + 1) * 8)); CK(tmp.get(&d_err, 8));
    const unsigned long long err0 = ~0ull;
    CK(cudaMemcpyAsync(d_off, off.data(), (size_t)(G + 1) * 8, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(d_err, &err0, 8, cudaMemcpyHostToDevice, e->stream));
    Pinned pin;
    CK(cudaHostAlloc(&pin.p, 2 * half, cudaHostAllocDefault));
    Events ev;
    std::vector<std::array<cudaEvent_t, 3>> chunk_ev;
    cudaEvent_t copied[2] = {nullptr, nullptr};   // the H2D of the chunk last read into each pinned half
    int g0 = 0, k = 0;
    while (g0 < G) {
        int g1 = g0;
        while (g1 < G && (size_t)(off[g1 + 1] - off[g0]) * 4 <= half) ++g1;
        const int buf = k & 1;
        const size_t bytes = (size_t)(off[g1] - off[g0]) * 4;
        if (copied[buf]) CK(cudaEventSynchronize(copied[buf]));
        const double t0 = now_s();
        if (!R.raw((uint8_t *)pin.p + buf * half, bytes)) return snap_bad(P, "truncated");
        g_snap_sec[3] += now_s() - t0;
        std::array<cudaEvent_t, 3> ce{ev.make(), ev.make(), ev.make()};
        CK(cudaEventRecord(ce[0], e->stream));
        CK(cudaMemcpyAsync(d_stage + buf * half, (uint8_t *)pin.p + buf * half, bytes, cudaMemcpyHostToDevice, e->stream));
        CK(cudaEventRecord(ce[1], e->stream));
        k_snap_unpack<<<std::min(e->gc_pool_main, g1 - g0), GC_THREADS, 0, e->stream>>>(A, g0, g1, d_off, off[g0], (const uint32_t *)(d_stage + buf * half), d_err);
        CK(cudaGetLastError());
        CK(cudaEventRecord(ce[2], e->stream));
        chunk_ev.push_back(ce);
        copied[buf] = ce[1];
        g0 = g1; ++k;
    }
    unsigned long long err = 0;
    CK(cudaMemcpyAsync(&err, d_err, 8, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    for (auto &ce : chunk_ev) {
        float a = 0.f, b = 0.f;
        cudaEventElapsedTime(&a, ce[0], ce[1]); cudaEventElapsedTime(&b, ce[1], ce[2]);
        g_snap_sec[4] += a * 1e-3; g_snap_sec[5] += b * 1e-3;
    }
    if (err != ~0ull) {
        static const char *why[] = {"", "checksum mismatch", "header or size inconsistent", "free lists malformed", "index out of range"};
        const unsigned reason = (unsigned)(err & 0xffu);
        return snap_bad(P, "game " + std::to_string(err >> 8) + ": " + why[reason >= 1 && reason <= 4 ? reason : 0]);
    }
    if (!R.raw(hdr, 8) || !R.raw(&nbytes, 8) || hdr[0] != F_END || hdr[1] != 0u || nbytes != 0) return snap_bad(P, "truncated (no end mark)");
    guard.e = nullptr;
    *out = e;
    return B200_OK;
}
