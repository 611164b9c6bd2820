/*
 * b200_tetris_mcts.h — C-ABI of the B200-native batched Tetris-MCTS engine (libb200_tetris_mcts.so).
 *
 * This is the drop-in boundary for the reference's per-move simulation loop.  Every entry point names the
 * reference interface it replaces (file:line in hrpan/tetris_mcts @ 7f24f8d).  Conventions:
 *   - extern "C", plain pointers and sizes, no C++/torch types; the caller owns every buffer it passes;
 *   - pointers are HOST pointers unless the name says `_dev`;
 *   - every function returns 0 on success or a B200_ERR_* code; b200_last_error() gives the text;
 *   - one host thread per engine; all work of an engine is issued on ONE CUDA stream: its own, or the caller's (b200_engine_set_stream);
 *   - there is no CPU fallback: without a CUDA device every compute entry point returns B200_ERR_CUDA.
 * Games travel as the 80-byte packed record of SPEC_PYTETRIS.md §6 (20 uint32 words).
 */
#ifndef B200_TETRIS_MCTS_H
#define B200_TETRIS_MCTS_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_ERR_BAD_ARG 1
#define B200_ERR_CUDA 2
#define B200_ERR_ARENA_FULL 3   /* reference: "MAX_NODES EXCEEDED" then UB, agents/cppmodule/agent.cpp:227-231 */
#define B200_ERR_TRACE_FULL 4
#define B200_ERR_NO_WEIGHTS 5

#define B200_REC_WORDS 20
#define B200_KEY_WORDS 12
#define B200_N_ACTIONS 7        /* agents/cppmodule/core.h:17 */
#define B200_N_WEIGHTS 478342   /* model/model_vv.py:13-46 Net: state_dict order, PyTorch layouts, + out_ubound, out_lbound */

enum { B200_MODE_LP = 0,        /* agents/ValueSimLP.py:13-70 */
       B200_MODE_SINGLE = 1,    /* agents/ValueSim.py:52-94 */
       B200_MODE_VANILLA = 2,   /* agents/Vanilla.py:17-64 */
       B200_MODE_DIST = 3 };    /* agents/core_distributional.py:82-124 driven as agents/DistValueSimOnline.py:36-75 sketches */
enum { B200_EVAL_SYNTHETIC = 0, /* test evaluator (hash of the observation), shared with the CPU oracle */
       B200_EVAL_NET = 1,       /* model/model_vv.py Model_VV.inference, fp32 CUDA cores.  Takes finite weights of any size, so a sum can
                                   overflow fp32 to +-inf, and inf - inf gives NaN.  The value network's ReLU is fmaxf, and fmaxf(NaN, 0)
                                   is 0 where torch's relu keeps the NaN: such a board gets finite (and wrong) v and var where the fp32
                                   reference returns NaN.  The distributional network's LeakyReLU keeps NaN (DESIGN §5). */
       B200_EVAL_NET_TC = 2,    /* same network on wgmma tensor cores (fp16 x 2 operand split, 3 products per product); in B200_MODE_DIST:
                                   model/model_distributional.py on tensor cores (csrc/distnet_tc.cuh) instead of the fp32 CUDA-core kernels */
       B200_EVAL_NET_FP16 = 3,  /* same weights and tensor-core kernels as B200_EVAL_NET_TC with ONE fp16 term per operand and one product per
                                   product (about 1/3 of the MMA work).  Every activation and conv / fc1 weight is rounded to fp16 (2^-11
                                   relative) instead of split (2^-22), so outputs are NOT within 1e-5 of Model_VV: DESIGN §5 states
                                   the bounds (act3 per element within 2^-10 of the board's largest |term| sum, v and var within
                                   2^-11 relative plus two ill-conditioned cases); the search on those outputs is exact.  Same weight
                                   limits as B200_EVAL_NET_TC.  Not available in B200_MODE_DIST (b200_engine_create returns
                                   B200_ERR_BAD_ARG) nor for b200_load_dist_weights. */
       B200_EVAL_DIST_FP16 = 4, /* model/model_distributional.py on the tensor-core kernels of B200_EVAL_NET_TC in B200_MODE_DIST, with ONE
                                   fp16 term per operand and one product per product (about 1/3 of the MMA work).  Every conv activation
                                   and conv / fc1 weight is rounded to fp16 (2^-11 relative), so the probabilities are NOT within 1e-5 of
                                   the fp32 network: DESIGN §5 states the bounds (act2 per element within 2^-10 of the board's largest
                                   |term| sum plus a floor, probabilities within 2 e_z p); the search on those outputs is exact.  Valid
                                   only in B200_MODE_DIST (b200_engine_create returns B200_ERR_BAD_ARG otherwise: net_fp16 is the value
                                   network's one-term kind); b200_load_weights returns B200_ERR_BAD_ARG (no value network);
                                   b200_load_dist_weights takes the weight limits of B200_EVAL_NET_TC. */
       B200_EVAL_EXTERNAL = 5,  /* the caller's evaluator (OnlineMCTSAgent(..., evaluator=, evaluation_type=0), agents/cppmodule/agent.cpp:
                                   423-436; ValueSimLP.mcts' self.model.inference, agents/ValueSimLP.py:55-60): each simulation step is driven
                                   with b200_ext_step_begin / b200_ext_step_end below.  B200_MODE_LP, B200_MODE_SINGLE and B200_MODE_DIST
                                   (b200_engine_create returns B200_ERR_BAD_ARG in B200_MODE_VANILLA, whose evaluator is the rollout). */
       B200_EVAL_EXTERNAL_GAME = 6 }; /* the caller's leaf-GAME evaluator (MCTSAgent(..., evaluator, evaluation_type=1), agent.cpp:449-455;
                                   VanillaC's random_playout): in place of the rollout, each step hands the expanded leaf of every game as a
                                   packed record to the caller, whose (value, variance) is backed up as it is (value not added to the leaf's
                                   score, variance in place of rollout_variance).  Driven with b200_ext_step_begin(B200_BOARD_RECORD) /
                                   b200_ext_step_end.  B200_MODE_VANILLA only (b200_engine_create returns B200_ERR_BAD_ARG otherwise).
                                   Counter 5 (rollout steps) stays 0; counter 2 counts the leaves handed out. */

typedef struct b200_engine b200_engine;

typedef struct {
    int32_t n_games;            /* concurrent, independent game trees */
    int32_t max_nodes;          /* per-game arena, agents/agent.py:36 / agents/ValueSim.py:16 */
    int32_t mode;               /* B200_MODE_* */
    int32_t low;                /* check_low threshold: 1 (ValueSimLP.py:27), 5 (Vanilla.py:27) */
    int32_t lp_end_from_obs;    /* 0: ValueSimLP.py:25 behaviour; 1: agent.cpp:538 */
    int32_t lp_var_gamma2;      /* 1: core.h:365; 0: agent.cpp:558 */
    int32_t stale_pop;          /* 1: reproduce agents/agent.py:229-232 literally */
    int32_t overflow_reset;     /* 0: arena full after GC is an error (reference: IndexError agent.py:99 / UB agent.cpp:227-231);
                                   1: drop that game's tree and re-root it at the live game (counter 7 counts these) */
    int32_t eval_kind;          /* B200_EVAL_* */
    int32_t trace_max;          /* longest root-to-leaf path stored (0 -> 512) */
    int32_t actions_per_drop, scoring, randomizer;   /* play.py:75 env_args */
    int32_t device;             /* CUDA device ordinal */
    uint32_t seed;              /* search RNG stream base (replaces libc rand(), core.h:62,76, and random.randint, Vanilla.py:52) */
    double gamma;               /* ValueSim.py:14 0.999 / Vanilla.py:9 0.99 */
    double rollout_variance;    /* Vanilla.py:54 1e3 / VanillaC.py:8 1e5 */
    int32_t dist_bins;          /* B200_MODE_DIST: atoms, DistValueSimOnline.py:13 (50) */
    double dist_vmin, dist_vmax;   /* value range, DistValueSimOnline.py:13 (0, 5000) */
} b200_config;

const char *b200_last_error(void);
int b200_device_count(void);

/* --- engine lifetime: replaces TreeAgent.__init__/init_array (agents/agent.py:36-88), Agent.close (:303-307) */
int b200_engine_create(const b200_config *cfg, b200_engine **out);
int b200_engine_destroy(b200_engine *e);
/* --- SURVEY 8(b).5 "explicit cudaStream_t" (no reference counterpart: the reference is synchronous CPU code).  cuda_stream is a
 *     cudaStream_t passed as void* so that this header needs no CUDA include: from now on ALL work of the engine (kernels, the captured
 *     simulation step, async copies, the event timers) is issued on it; NULL = a private non-blocking stream again (the default).  The
 *     engine drains its previous stream inside the call; the caller owns its stream.  The legacy default stream cannot be captured into
 *     a CUDA graph: with it the step falls back to direct launches.  b200_engine_get_stream returns the stream in use, so that a caller
 *     that produces or consumes `_dev` buffers on its own stream can order against it (cudaStreamWaitEvent). */
int b200_engine_set_stream(b200_engine *e, void *cuda_stream);
int b200_engine_get_stream(b200_engine *e, void **cuda_stream_out);

/* --- Model.load (model/model.py:163-174): weights = the state_dict tensors concatenated (B200_N_WEIGHTS floats).
 *     A B200_EVAL_NET_TC or B200_EVAL_NET_FP16 engine returns B200_ERR_BAD_ARG, keeping its previous weights, when a conv or fc1 weight
 *     is non-finite or has |w| * 64 > 65504 (fp16 overflow in the tensor cores' scaled operands); the same holds for
 *     b200_load_dist_weights (B200_EVAL_NET_TC, B200_EVAL_DIST_FP16). */
int b200_load_weights(b200_engine *e, const float *weights);

/* --- snapshot (no reference counterpart: the reference checkpoints the model only).  b200_engine_save writes everything a later call can
 *     read to `path`: every b200_config field, the path-cache / deep-lane / gc_headroom settings, the weights as b200_load_weights /
 *     b200_load_dist_weights took them, the counters and the finished-games log, the replay memory with its policy (the std::mt19937 and
 *     the trimming sampler included), and each game's arena packed on the device to its live slots, free lists, records, table entries and
 *     last trace, with a 64-bit checksum per game (DESIGN §4c).  The image streams through a bounded staging buffer: two halves of
 *     max(b200_snapshot_set_staging / 2, the largest packed game) bytes in device memory and the same again in pinned host memory, so
 *     64 MB of each (128 MB in all) by default.  It is
 *     written to path + ".tmp", flushed, synced and renamed: an interrupted save leaves a previous image at `path` intact.  *bytes_out
 *     (may be NULL) = the file's size.  A step open between b200_ext_step_begin and _end returns B200_ERR_BAD_ARG.
 *   b200_engine_load creates an engine from such an image (device -1: the saved ordinal) that continues bit for bit as the saved one
 *     would have: the same actions, statistics, arenas, counters, memory and policy draws.  The path cache restarts empty (it changes no
 *     result).  A truncated or corrupted file, a wrong magic or format version, or an unknown field returns B200_ERR_BAD_ARG with the
 *     reason in b200_last_error and leaves nothing allocated.  The checksums detect corruption; an image is not authenticated.
 *   b200_snapshot_timing: seconds of this thread's last save {device pack, D2H, write} and load {read, H2D, device unpack}. */
int b200_engine_save(b200_engine *e, const char *path, int64_t *bytes_out);
int b200_engine_load(const char *path, int device, b200_engine **out);
int b200_snapshot_set_staging(int64_t bytes);   /* process-wide; <= 0: the default */
int b200_snapshot_timing(double *sec6);

/* --- TreeAgent.update_root (agents/agent.py:296-301) for all games: recs[n_games][20] */
int b200_set_games(b200_engine *e, const uint32_t *recs);
int b200_get_games(b200_engine *e, uint32_t *recs);
int b200_update_root(b200_engine *e, int auto_reset);

/* --- TreeAgent.remove_nodes (agents/agent.py:246-257; a public method, also reached from new_node :96-97 when the free list is
 * empty): collect every game that has fewer than min_free free node slots (INT_MAX: every game), as one batched launch.
 * b200_set_gc_headroom(n > 0) makes b200_update_root / b200_play_move do that after re-rooting (the driver calling remove_nodes() between
 * moves whenever len(agent.available) < n; b200_set_games only re-roots); 0 (default) = only the reference's own call site, inside new_node. */
int b200_remove_nodes(b200_engine *e, int min_free);
int b200_set_gc_headroom(b200_engine *e, int min_free);

/* --- scheduling only (no reference counterpart, no effect on any result): the up to max_games games whose last trace was longest walk the tree
 * on a second stream, so that a simulation step of the other games does not last as long as the deepest walk of all (ValueSim / ValueSimLP with
 * B200_EVAL_NET_TC or B200_EVAL_NET_FP16; ignored otherwise).  0 (default) = one lane. */
int b200_set_deep_lane(b200_engine *e, int max_games);

/* --- memory traffic only (no reference counterpart, no effect on any result): the PATH CACHE.  Consecutive simulations of a game walk almost
 * the same root-to-leaf path (select_trace_obs, core.h:167-224, restarts at the root every time); with the cache on, a walk leaves next to its
 * trace the row fields and the children's statistics of every level, the backup (core.h:226-381) refreshes the copies it changes and drops
 * the ones a transposition made stale, and the next walk serves every level that is still valid from one sequential line instead of two
 * dependent random accesses.  B200_MODE_LP with max_nodes <= 65536; 192 bytes x trace_max per game (entry 160 + own record 16 + child ids 16).  0 (default) = off. */
int b200_set_path_cache(b200_engine *e, int on);

/* --- TreeAgent.mcts (agents/ValueSimLP.py:13, ValueSim.py:52, Vanilla.py:17): `sims` simulations on every game */
int b200_run_sims(b200_engine *e, int sims);

/* --- the caller's evaluator (B200_EVAL_EXTERNAL, B200_EVAL_EXTERNAL_GAME): one simulation step of every game in two halves around the
 *   caller's network or leaf-game function.
 *   b200_ext_capacity: max_rows = the most rows one step hands out (7 * n_games in B200_MODE_LP, n_games otherwise); out_cols = 2 (v, var),
 *     or dist_bins in B200_MODE_DIST.
 *   b200_ext_step_begin: select + expand and the collections of one step (the code b200_run_sims runs), then this step's evaluation
 *     requests as boards: boards_dev (DEVICE) [max_rows][200] = NCHW [n,1,20,10] in {-1, 0, 1} as Model_VV.inference sees them (the
 *     board bits, the four falling-piece cells -1), int8 (B200_BOARD_INT8) or float32 (B200_BOARD_F32); ids_dev (DEVICE, may be NULL)
 *     [max_rows] = game * 8 + slot of each row (slot = child index in LP, 7 = the leaf itself).  Rows are in ascending (game, slot) order,
 *     so the batch is a function of the search state alone, not of the order the device queued the requests in.  Synchronises the
 *     engine's stream and returns *n_rows (0 is possible, e.g. when every leaf is a game over).  In LP the rows are the unique children
 *     whose observation has no statistics yet; the reference also evaluates the others and discards those outputs (core.h:303-381), so
 *     the results are the same.
 *   b200_ext_step_end: out_dev (DEVICE) [n_rows][out_cols] fp32 row-major (stored as they are, NaN included), then the backup.
 *     Asynchronous on the engine's stream, like b200_run_sims: order the evaluator's work against b200_engine_get_stream.
 *   Between the two a step is open: a second step_begin, and b200_run_sims, b200_play_move, b200_update_root, b200_set_games,
 *   b200_env_step, b200_remove_nodes, b200_set_path_cache, b200_engine_set_stream and the b200_replay_* calls return B200_ERR_BAD_ARG;
 *   step_end without an open step too.  Reading calls (b200_export_game, b200_export_dist, b200_get_stats, b200_counters, b200_status)
 *   work as usual.  An external engine returns B200_ERR_BAD_ARG from b200_run_sims, b200_play_move, b200_load_weights,
 *   b200_load_dist_weights, b200_valuenet_forward, b200_distnet_forward and the b200_debug_* network readers; b200_set_deep_lane is
 *   ignored; counter 12 is the longest trace since the engine was created (only b200_run_sims resets it).  The kernels of the split
 *   count under phase 6 of b200_phase_ms. */
/*   B200_EVAL_EXTERNAL_GAME: max_rows = n_games, out_cols = 2.  b200_ext_step_begin takes board_dtype B200_BOARD_RECORD (the only dtype it
 *     takes; an external engine refuses it) and writes into boards_dev (DEVICE, 16-byte aligned) uint32 [n_games][20] the packed record
 *     (SPEC_PYTETRIS §6) of the leaf of every game whose step expanded one (the games the rollout would play out), in ascending game
 *     order; ids_dev[row] = the game.  b200_ext_step_end takes [n_rows][2] fp32 (value, variance) per row. */
#define B200_BOARD_INT8 0
#define B200_BOARD_F32 1
#define B200_BOARD_RECORD 2
int b200_ext_capacity(b200_engine *e, int32_t *max_rows, int32_t *out_cols);
int b200_ext_step_begin(b200_engine *e, void *boards_dev, int board_dtype, int32_t *ids_dev, int32_t *n_rows);
int b200_ext_step_end(b200_engine *e, const float *out_dev);

/* --- TreeAgent.compute_stats / get_action (agents/agent.py:153-185): stats[n][3][7], action[n] */
int b200_get_stats(b200_engine *e, float *stats, int32_t *action);

/* --- Tetris.play on the engine's live games (play.py:150): actions[n]; NULL = the argmax actions of the last stats */
int b200_env_step(b200_engine *e, const int32_t *actions);

/* --- one whole move of play.py:118-177 for every game: mcts -> get_action -> play -> update_root (-> reset) */
int b200_play_move(b200_engine *e, int sims, int auto_reset, int32_t *actions_out, float *stats_out);

/* --- the episodes that ended inside b200_update_root(auto_reset) / b200_play_move since the last call (play.py:161-177 prints
 *     `Episode: .. Score: .. Lines Cleared: ..` from these numbers before game.reset()): out4[i] = {game, score, line_clears, episode};
 *     at most cap rows are copied, *count_out = episodes ended (the device log holds 4 * n_games rows between drains) */
int b200_finished_games(b200_engine *e, int32_t *out4, int cap, int32_t *count_out);

int b200_status(b200_engine *e, int32_t *status);            /* per-game 0 ok / B200_ERR_ARENA_FULL / B200_ERR_TRACE_FULL */
int b200_counters(b200_engine *e, uint64_t *out16);          /* 0 sims 1 expansions 2 eval requests 3 gcs 4 trace levels
                                                                5 rollout steps 6 new nodes 7 tree resets 8 games finished 9 score sum 10 lines sum
                                                                12 longest trace of the last b200_run_sims (not cumulative)
                                                                13 trace levels served by the path cache (of counter 4) */
int b200_sync(b200_engine *e);
int b200_timer_start(b200_engine *e);                        /* CUDA-event stopwatch on the engine's stream (sync, then record) */
int b200_timer_stop(b200_engine *e, float *ms);              /* record, wait, elapsed milliseconds since b200_timer_start */
int b200_set_timing(b200_engine *e, int on);                 /* CUDA-event timing of each phase on the engine's stream */
int b200_phase_ms(b200_engine *e, float *ms8, uint64_t *launches8);   /* 0 select+expand 1 conv 2 fc 3 backup 4 rollout 5 synth 6 stats/step/root 7 gc+resume */

/* --- the arena of one game in the reference's array layout (agents/agent.py:58-88); any pointer may be NULL */
int b200_export_game(b200_engine *e, int game, int32_t *child, float *score, int32_t *episode, int32_t *n2o,
                     int32_t *visit, float *value, float *variance, uint8_t *obs_end, uint32_t *game_recs,
                     uint32_t *obs_keys, int32_t *root, int32_t *last_trace, int32_t *last_trace_len);

/* --- Model_VV.inference (model/model_vv.py:210-217): states[k][200] int8 -> v[k], var[k] */
int b200_valuenet_forward(b200_engine *e, const int8_t *states, int k, float *v, float *var);

/* --- pyTetris.Tetris ctor / reset / play / getState for host-resident games (play.py:75-76,150,169,
 *     agents/agent.py:116).  b200_tetris_new: reset == 0 builds n fresh games (seeds[n] or NULL = default seed),
 *     reset != 0 applies Tetris.reset() to the n records in place (keeps each RNG stream, SPEC §4). */
int b200_tetris_new(uint32_t *recs, int n, int actions_per_drop, int scoring, int randomizer, const uint32_t *seeds, int reset);
int b200_tetris_step(uint32_t *recs, const int32_t *actions, int n);
int b200_tetris_state(const uint32_t *recs, int8_t *out, int n);
/* --- the same on DEVICE records owned by the caller (e.g. the leaf games of B200_EVAL_EXTERNAL_GAME), for a leaf evaluator that runs at
 *     device speed.  Unlike the engine's `_dev` calls these are ASYNCHRONOUS: each only enqueues its kernel on `stream` (a cudaStream_t
 *     passed as void*; NULL = the legacy default stream) and returns; order the caller's work against that stream.  recs_dev is
 *     uint32 [n][20], 16-byte aligned; n = 0 is a no-op.  No engine is involved.
 *   b200_tetris_step_dev: one Tetris.play per record, in place; action ids outside 0..6 move nothing (SPEC §3: gravity still ticks).
 *   b200_tetris_state_dev: getState() as int8 (B200_BOARD_INT8) or float32 (B200_BOARD_F32) [n][1][20][10]: the board bits and -1 on the
 *     four falling-piece cells, the boards B200_EVAL_EXTERNAL hands out.
 *   b200_tetris_playout_dev: random playouts (the rollout's loop): row i plays xorshift32(rng_dev[i]) % n_actions (1..8; 8 includes the
 *     no-op 7, VanillaC's randint(0, 7)) until its game is over or after max_steps (>= 0) actions.  The final record and stream are written
 *     back (a stream of 0 starts as 0x2545F491); steps_dev[i] (may be NULL) = the actions played. */
int b200_tetris_step_dev(uint32_t *recs_dev, const int32_t *actions_dev, int n, void *stream);
int b200_tetris_state_dev(const uint32_t *recs_dev, void *out_dev, int dtype, int n, void *stream);
int b200_tetris_playout_dev(uint32_t *recs_dev, uint32_t *rng_dev, int n, int n_actions, int max_steps, int32_t *steps_dev, void *stream);

/* --- single-call twins of agents/cppmodule/core.cpp:20-26 on the reference's own arrays (mutated in place) */
int b200_select_trace_obs(int index, const int32_t *child, const int32_t *visit, const float *value,
                          const float *variance, const float *score, const int32_t *n_to_o, int M, int low,
                          uint32_t *rng_state, int32_t *trace_out, int max_trace, int32_t *trace_len);
int b200_backup_trace_obs(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                          const int32_t *n_to_o, const float *score, int M, double v, double var, double gamma);
int b200_backup_trace_obs_LP(const int32_t *trace, int D, int32_t *visit, float *value, float *variance,
                             const int32_t *n_to_o, const float *score, const uint8_t *end, int M,
                             const int32_t *c_nodes, const int32_t *c_obs, int k, const float *v, const float *var,
                             double gamma, int mixture, int averaged);
/* test aid: the walk's z(n) for n[count] (host table below 65536, evaluated on the device above; DESIGN §3 states the exact range) */
int b200_debug_ztab(const int32_t *n, int count, float *out);
int b200_get_unique_child_obs(int index, const int32_t *child, const float *score, const int32_t *n_to_o, int M,
                              int32_t *c_nodes, int32_t *c_obs, int32_t *k_out);
int b200_get_all_childs(int index, const int32_t *child, int M, uint8_t *mark);

/* --- distributional cores (agents/core_distributional.py, BASELINE config 5), operator level, reference array layout:
 *     node_stats f32[M][5] = {visit, mean, reward, variance, M2}, node_dist f32[M][bins], child int32[M][7] */
int b200_dist_shift_distribution(const float *dist, int bins, double x, double vmin, double vmax, float *out);     /* :12-36, x >= 0 */
int b200_dist_mean_variance(const float *dist, int bins, double vmin, double vmax, double *mean, double *var);     /* :48-63 */
int b200_dist_select_trace(int index, const int32_t *child, const float *node_stats, int M, int low, uint32_t *rng_state,
                           int32_t *trace_out, int max_trace, int32_t *trace_len);                                 /* :82-106 */
int b200_dist_backup_trace(const int32_t *trace, int D, float *node_stats, float *node_dist, int M, int bins, double r,
                           const float *dist, double vmin, double vmax);                          /* :109-124, bins <= 64 */

/* --- distributional engine (B200_MODE_DIST): Model.load / Model.inference of model/model_distributional.py:18-57 and the
 *     node-indexed arrays of one game.  weights: seq.conv1.w[32,1,4,4] b[32] seq.conv2.w[32,32,4,4] b[32] seq.fc1.w[128,2048]
 *     b[128] seq.fc_v.w[atoms,128] b[atoms] concatenated (the reference hard-codes a 22x10 input, model_distributional.py:27:
 *     the 20x10 observation gets two empty rows on top). */
int b200_load_dist_weights(b200_engine *e, const float *weights, int atoms);
int b200_distnet_forward(b200_engine *e, const int8_t *states, int k, int atoms, float *dist);
/* test aid: the conv stack's output of the tensor-core distributional network (B200_EVAL_NET_TC or B200_EVAL_DIST_FP16; other kinds
 * return B200_ERR_BAD_ARG) on states[k][200]: out[k][2048] in torch flatten order c*64 + y*4 + x, as the tensor cores' fp16 operands hold it */
int b200_debug_dist_act2(b200_engine *e, const int8_t *states, int k, float *out);
/* test aid: one layer of a tensor-core network exactly as the next layer reads it, from a forward pass on states[k][200].  dist = 0: the
 * value network (B200_EVAL_NET_TC or B200_EVAL_NET_FP16), layer 1..3 = act1 [32][18][8], act2 [32][16][6], act3 [32][14][4]; dist = 1: the
 * distributional network (B200_EVAL_NET_TC or B200_EVAL_DIST_FP16), layer 1..2 = act1 [32][19][7], act2 [32][16][4].  out[k][nt][...] holds
 * fp16 term s < nt of each element divided by 16 (nt = 2 for net_tc, 1 for the fp16 kinds).  layer 4 (value) / 3 (distributional): fc1's
 * raw fp32 accumulator, out[k][256] / out[k][128] in torch column order (the value before the 2^-10, the bias and the activation).
 * layer 0: the same pass's outputs, out[k][2] = (v, var) or out[k][atoms] = probabilities. */
int b200_debug_tc_acts(b200_engine *e, int dist, const int8_t *states, int k, int layer, float *out);
/* test aid: every stage of an fp32 CUDA-core network (B200_EVAL_NET only; other kinds, dist not 0 / 1 or a layer outside 0..4 return
 * B200_ERR_BAD_ARG, a network without weights B200_ERR_NO_WEIGHTS) exactly as the kernels computed it, from one forward pass on
 * states[k][200].  dist = 0, the value network: layer 0 = (v, var) out[k][2], 1 = act1 [32][18][8], 2 = act2 [32][16][6], 3 = act3
 * [32][14][4] (the production buffer fc1 reads), 4 = fc1's fp32 accumulator out[k][256] in torch column order (before the bias and the
 * ReLU).  dist = 1, the distributional network: layer 0 = probabilities out[k][atoms], 1 = act1 [32][19][7], 2 = act2 [32][16][4] (the
 * production buffer), 3 = fc1's accumulator out[k][128] (bias included, before the LeakyReLU), 4 = the logits out[k][atoms]. */
int b200_debug_net_acts(b200_engine *e, int dist, const int8_t *states, int k, int layer, float *out);
/* test aid: the production backup (k_backup, launched as b200_run_sims launches it) on a tree in the reference's layout (agents/agent.py:58-88),
 * on a one-game engine of mode lp, single or vanilla (others, or more games, return B200_ERR_BAD_ARG).  child[M][7], n_to_o[M], score[M] per
 * node; visit / value / variance / end[M] per observation (the first three updated in place); trace[D] (D <= trace_max); leaf_kind 0 = terminal,
 * 1 = expanded; eval_out[8][2] = (value, variance) per child slot (LP) or of the leaf in slot 7 (single); rollout_val (vanilla).  Overwrites
 * the engine's tree of game 0 with the given one.  With the path cache on (and only then) pc_len points to the number of entries the walk left
 * valid (<= D - 1 after an expansion, <= D at a terminal leaf); they are filled from the given arena as the walk stores them, and pc_len, the
 * own records pc_own[D][4], the child ids pc_sib[D][8], the entries pc_ent[D][8][4] and pc_var[D][8] come back as the backup left them. */
int b200_debug_backup(b200_engine *e, int M, const int32_t *child, const int32_t *n_to_o, const float *score, int32_t *visit, float *value,
                      float *variance, const uint8_t *end, const int32_t *trace, int D, int leaf_kind, const float *eval_out, float rollout_val,
                      int32_t *pc_len, int32_t *pc_own, uint16_t *pc_sib, int32_t *pc_ent, int32_t *pc_var);
/* test aid: game `game` of an engine of mode lp, single or vanilla set to a tree in the reference's layout (child[M][7], n_to_o / score per
 * node, visit / value / variance / end per observation), as expansions would have left it: link words by the production finish_expansion,
 * root, the game's check_low stream (rng_state != 0), status ok, an empty path cache, and the game-over bit set exactly on the nodes without
 * children, so that b200_run_sims runs the production walk and terminal backup on it.  b200_debug_game_state reads the stream back with the
 * path cache's valid length (0 with the cache off). */
int b200_debug_load_tree(b200_engine *e, int game, int M, const int32_t *child, const int32_t *n_to_o, const float *score, const int32_t *visit,
                         const float *value, const float *variance, const uint8_t *end, int root, uint32_t rng_state);
int b200_debug_game_state(b200_engine *e, int game, uint32_t *rng_state, int32_t *pc_len);
int b200_export_dist(b200_engine *e, int game, float *node_stats /* [M][5] */, float *node_dist /* [M][bins] */);

/* --- replay samples of the live search (ValueSim.store_nodes, agents/ValueSim.py:122-159): observations with
 *     visit >= min_visits and not end, packed as {int8 state[200], f32 value, f32 variance, f32 visit} = 212 B.
 *     out_dev is a DEVICE buffer of capacity*212 bytes (e.g. a torch tensor handed to the NCCL all-gather). */
int b200_collect_samples_dev(b200_engine *e, int min_visits, void *out_dev, int capacity, int32_t *count_out);

/* --- online replay memory (ValueSim.memory agents/ValueSim.py:14-37; OnlineMCTSAgent agent.cpp:588-617): when enabled, every
 *     garbage collection appends the observations it frees that have visit >= min_visits and are not `end`
 *     (store_nodes, ValueSim.py:122-159 / agent.cpp:777-819) until `capacity` rows are held.  b200_replay_drain_dev copies the
 *     rows to a DEVICE buffer (trainer input / NCCL all-gather block) and empties the memory (ValueSim.py:183). */
int b200_replay_enable(b200_engine *e, int min_visits, int capacity);
int b200_replay_drain_dev(b200_engine *e, void *out_dev, int capacity, int32_t *count_out);

/* --- the online agent's accumulation policies and memory trimming (OnlineMCTSAgent::remove_nodes agent.cpp:619-708: policies 0-3;
 *     weighted_trimming :710-749; random_trimming :751-775; store_nodes' random drop :800-801), on the memory b200_replay_enable created
 *     (memory_size = capacity, min_visit = min_visits).  b200_replay_policy_step = the decision the reference takes inside remove_nodes() after
 *     storing: call it after collections (single game: after every step / update_root in which counter 3 moved — then memory contents, trimming
 *     and the moments of training equal the compiled agent.cpp's; batched: once per move) with current_episode = games finished so far
 *     (agent.cpp:279-280).  *train_now != 0: train on the first *memory_index rows (b200_replay_peek_dev), then b200_replay_policy_trained. */
int b200_replay_policy(b200_engine *e, int accumulation_policy, int episodes_per_train, int memory_growth_rate);
int b200_replay_policy_step(b200_engine *e, int64_t current_episode, int32_t *train_now, int32_t *memory_index);
int b200_replay_policy_trained(b200_engine *e, int64_t current_episode);
int b200_replay_peek_dev(b200_engine *e, void *out_dev, int n_rows);
int b200_replay_append(b200_engine *e, const uint8_t *rows_host, int n_rows);   /* rows join the memory as a collection's would: in order, until it is full */
int b200_replay_append_dev(b200_engine *e, const void *rows_dev, int n_rows);   /* the same from a DEVICE buffer (e.g. rows all-gathered from other ranks) */

/* --- value-network training step (SURVEY 8f.2): Model_VV._loss / Model.train / Yogi.step / Model_VV.train_data of the reference
 *     (model/model_vv.py:94-153,227-231, model/model.py:52-119, model/yogi.py:39-90) on the device.  weights = the state_dict vector of
 *     b200_load_weights (PyTorch layouts); a batch is {states int8[n][200], value f32[n], variance f32[n], weight f32[n]} (the four arrays
 *     of ValueSim.memory, agents/ValueSim.py:25-30).  Host logic that stays on the host (validation split, early stopping, checkpoint files):
 *     tetris_mcts_b200/model/model_vv.py Model_VV.train_data (host arrays) and Model_VV.train_rows (device replay rows, batches drawn on the
 *     device by b200_trainer_train_rows_dev). */
typedef struct b200_trainer b200_trainer;
const char *b200_trainer_last_error(void);
int b200_trainer_create(int device, const float *weights, int max_batch, b200_trainer **out);     /* Model_VV._init_model (model_vv.py:125-134) */
/* Trainer kinds: which GEMMs a training step's contractions run on.  Every b200_trainer_* entry point below works on either kind with the
 * same contract; b200_trainer_create is b200_trainer_create_kind(..., B200_TRAIN_FP64, ...).
 *   B200_TRAIN_FP64  CUDA-core GEMMs accumulating in fp64, rounded once to fp32.
 *   B200_TRAIN_TC    the conv / fc1 forward, input-gradient and weight-gradient GEMMs on Hopper tensor cores (3xTF32: each fp32 operand
 *                    split into two tf32 terms, three wgmma products accumulated in fp32, fp32 chains capped at 2048 k with fp64 partials
 *                    summed in a fixed order).  Loss, gradient norm and each gradient tensor stay within 1e-5 (relative, resp. of the
 *                    tensor's norm) of float64 arithmetic; fp32's exponent range is kept, so small gradients do not flush.  Bit-
 *                    reproducible run to run, and train_rows_dev stays bit-identical to step_rows_dev fed the same indices, as for fp64.
 *   B200_TRAIN_TF32  the same GEMMs on tensor cores with one tf32 term per operand (rna_tf32(x), |x - rna_tf32(x)| <= 2^-11 |x|): one
 *                    wgmma per k8 instead of three, and the tc kind's accumulation (32-k tiles, round-to-nearest chunk sums over <= 2048 k,
 *                    fp64 partials).  Per element: the exact products of the rounded operands, summed within tc's accumulation bound.
 *                    Against float64: each GEMM output lies within 2^-10 (two operand roundings of 2^-11) of its |term| sum plus tc's
 *                    accumulation (~1e-5), once per product on a result's path: the loss and loss_std stay within 4 * 2^-10 (four
 *                    forward products), the gradient norm within 8 * 2^-10.  Gradient elements sum over pixels whose terms cancel and
 *                    see the forward error through GaussianLL's mean - pred, so their bound is that error propagated through the
 *                    head and the backward pass in absolute values (tests/test_gpu_trainer_tf32.py error_bound; measured up to a few
 *                    percent of a tensor's norm, against 1e-5 for tc).  The convolutions are implicit GEMMs: conv1-3 gather their A operand from the NHWC activations (k =
 *                    ci*9 + ky*3 + kx), the conv weight gradients gather col^T the same way, and the input gradients of conv3 / conv2 are
 *                    one GEMM each, da[b][y][x][ci] = (act > 0) * sum over k = (ky*3 + kx)*32 + co (ascending, K = 288; taps outside
 *                    the output gradient are zero terms) of dY[b][y-ky][x-kx][co] * W[co][ci][ky][kx].  So a tf32 trainer has no
 *                    col1 / col2 / col3 / dcol3 / dcol2 buffers (355 392 B per sample of max_batch), and b200_trainer_debug_buffer
 *                    returns B200_ERR_BAD_ARG for those names.  Bit-reproducible, train_rows_dev == step_rows_dev, as the other kinds.
 * Weights and Yogi state mean the same in every kind, so a checkpoint of one kind loads into the others.
 * b200_trainer_create_kind returns B200_ERR_BAD_ARG for an unknown kind. */
#define B200_TRAIN_FP64 0
#define B200_TRAIN_TC 1
#define B200_TRAIN_TF32 2
int b200_trainer_create_kind(int device, const float *weights, int max_batch, int kind, b200_trainer **out);
int b200_trainer_destroy(b200_trainer *t);
int b200_trainer_set_hyper(b200_trainer *t, double lr, double beta1, double beta2, double eps, double weight_decay);   /* Yogi(...) model_vv.py:132 */
int b200_trainer_set_out_ubound(b200_trainer *t, float ub_value, float ub_variance);             /* model_vv.py:227-231 */
int b200_trainer_get_weights(b200_trainer *t, float *weights_out);                               /* model.state_dict() */
int b200_trainer_set_weights(b200_trainer *t, const float *weights);                             /* model.load_state_dict() */
int b200_trainer_get_state(b200_trainer *t, float *exp_avg, float *exp_avg_sq, int64_t *step);   /* optimizer.state_dict(); step -1 = no state yet */
int b200_trainer_set_state(b200_trainer *t, const float *exp_avg, const float *exp_avg_sq, int64_t step);   /* load_state_dict; step < 0 = reset_optimizer */
int b200_trainer_get_grads(b200_trainer *t, float *grads_out);                                   /* p.grad of the last step, state_dict order (478338 floats) */
/* test aid: a copy of one batch buffer as the last step / loss / step_rows_dev / grad_rows_dev left it, rows [0, n_rows) (fp32, row-major;
 * conv activations and their gradients NHWC [n][pixel][32], im2col buffers [n][pixel][ci*9 + ky*3 + kx]).  which: "x0" [200], "value",
 * "variance", "weight" [1], "col1" [144*9], "a1" [144*32], "col2" [96*288], "a2" [96*32], "col3" [56*288], "a3" [56*32], "flat" [1792]
 * (torch flatten order), "h" [256], "pred" [2], "lossv" [1], "dz" [2], "dh" [256], "dflat" [1792], "dc3" [56*32], "dcol3" [56*288],
 * "da2" [96*32], "dcol2" [96*288], "da1" [144*32]; or "d_sumsq": the last step's 10 per-tensor gradient sums of squares (double, n_rows
 * ignored).  Launches no kernel.  B200_ERR_BAD_ARG for an unknown name or n_rows outside [0, max_batch], and on a B200_TRAIN_TF32 trainer
 * for "col1", "col2", "col3", "dcol3" and "dcol2" (not allocated: its convolutions read the activations directly). */
int b200_trainer_debug_buffer(b200_trainer *t, const char *which, int n_rows, void *out);
/* Model_VV._loss under no_grad on one chunk (Model.compute_loss, model/model.py:52-83): mean and population std of (weight *) logl; pred_out NULL or [n][2] */
int b200_trainer_loss(b200_trainer *t, const int8_t *states, const float *value, const float *variance, const float *weight, int n,
                      int weighted, double *loss, double *loss_std, float *pred_out);
/* Model.train (model/model.py:95-119): forward, loss, backward, gradient norm, clip when grad_clip > 0, Yogi step */
int b200_trainer_step(b200_trainer *t, const int8_t *states, const float *value, const float *variance, const float *weight, int n,
                      int weighted, double grad_clip, double *loss, double *loss_std, double *grad_norm);
/* the same step on a batch gathered ON THE DEVICE from 212-byte replay rows (b200_replay_drain_dev / the all-gather block): idx[n] (host) are row
 * indices (np.random.choice, model/model.py:207), weight = visit * weight_scale (weights / weights.mean(), model/model.py:186-187) */
int b200_trainer_step_rows_dev(b200_trainer *t, const void *rows_dev, int n_rows, const int32_t *idx, int n, float weight_scale,
                               int weighted, double grad_clip, double *loss, double *loss_std, double *grad_norm);
/* Model.train_data's inner loop on device rows: `iters` steps of b200_trainer_step_rows_dev with batches of `batch` rows drawn ON THE DEVICE,
 * uniformly with replacement from rows [0, n_train_rows) (np.random.choice(n_train_rows, batch), model/model.py:207), and one host
 * synchronisation at the end.  Row i of step it (iteration number j = first_iter + it) is
 *     idx = splitmix64(splitmix64(splitmix64(seed) + j) + i) mod n_train_rows        (uint64 arithmetic, wrapping)
 *     splitmix64(x): z = x + 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9; z = (z ^ z >> 27) * 0x94D049BB133111EB; z ^ z >> 31
 * Gradient norm, clipping and Yogi are step_rows_dev's arithmetic: each step is bit-identical to b200_trainer_step_rows_dev fed those indices.
 * log_out (host): [iters][3] = {loss, loss_std, grad_norm} of each step. */
int b200_trainer_train_rows_dev(b200_trainer *t, const void *rows_dev, int n_train_rows, int batch, int iters, uint64_t seed, int64_t first_iter,
                                float weight_scale, int weighted, double grad_clip, double *log_out);
/* Model_VV._loss under no_grad on device rows [first, first + n) (a chunk of Model.compute_loss); *weight_sum = fp64 sum of visit * weight_scale */
int b200_trainer_loss_rows_dev(b200_trainer *t, const void *rows_dev, int first, int n, float weight_scale, int weighted,
                               double *loss, double *loss_std, double *weight_sum);
/* max(value), max(variance) and the fp64 sum of visits of device rows [0, n) (out_ubound, model_vv.py:227-231; the weight mean,
 * model/model.py:186-187), reduced in a fixed order on the trainer's stream */
int b200_rows_stats_dev(b200_trainer *t, const void *rows_dev, int n, float *max_value, float *max_variance, double *visit_sum);
/* --- data-parallel training: R ranks each compute the gradient of one slice of a batch, exchange the fp64 vectors and apply the same update.
 *     b200_trainer_set_stream: all later work of the trainer runs on the caller's stream (NULL: a private one again), so an exchange can be
 *       ordered on it without a host synchronisation.
 *     b200_trainer_grad_rows_dev: rows [lo, hi) of the batch b200_trainer_train_rows_dev draws for iteration `iter` (the same row formula, with
 *       the global row number i); forward, loss and backward on those rows with the gradient scaled by 1 / batch.  grad_dev (DEVICE) gets
 *       B200_TRAIN_VEC = 478338 + 3 doubles: the unrounded fp64 gradient (the values the fp32 gradient is rounded from) and the slice's
 *       {count, mean, M2} of (weight *) logl.  Asynchronous.  B200_ERR_BAD_ARG unless 0 <= lo < hi <= batch and hi - lo <= max_batch.
 *     b200_trainer_apply_grads_dev: parts_dev (DEVICE) = n_parts such vectors in rank order; g = (float)(((p0 + p1) + p2) + ...) element-wise,
 *       the loss moments joined in the same order, then train_rows_dev's gradient norm, clip and Yogi step; {loss, loss_std, grad_norm} go to
 *       device log slot log_slot.  Asynchronous.  One part covering the whole batch is bit-identical to a train_rows_dev step (weights,
 *       gradient, Yogi state, gradient norm; the loss may differ by reassociation).  Every rank applying the same parts holds the same bits.
 *     b200_trainer_read_log: synchronises and copies log slots [0, n) as [n][3] doubles. */
#define B200_TRAIN_VEC (478338 + 3)
int b200_trainer_set_stream(b200_trainer *t, void *cuda_stream);
int b200_trainer_grad_rows_dev(b200_trainer *t, const void *rows_dev, int n_train_rows, int batch, int lo, int hi, uint64_t seed, int64_t iter,
                               float weight_scale, int weighted, double *grad_dev);
int b200_trainer_apply_grads_dev(b200_trainer *t, const double *parts_dev, int n_parts, double grad_clip, int log_slot);
int b200_trainer_read_log(b200_trainer *t, int n, double *host);

#ifdef __cplusplus
}
#endif
#endif
