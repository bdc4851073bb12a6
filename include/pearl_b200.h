/* pearl_b200.h — C ABI of libpearlb200.so: the H100-native learner hot path of
 * facebookresearch/Pearl (`ReplayBuffer.sample -> PolicyLearner.learn()`).
 *
 * Conventions
 *   - extern "C", plain ints / pointers / sizes; no C++ or torch types.
 *   - every entry point returns 0 on success or a negative PRL_E* code; the
 *     message for the calling thread is available from prl_last_error().
 *   - the CALLER (PyTorch in pearl_b200/, or any other host) allocates and owns
 *     every device buffer; the library owns only its opaque handles, a pinned
 *     staging area for host pushes and small workspaces.  Pointers registered
 *     by *_create / *_bind stay referenced until *_destroy.
 *   - all device work is enqueued on the `stream` argument (a cudaStream_t
 *     passed as void*; NULL = legacy default stream).  No hidden
 *     synchronisation except where stated.
 *   - one handle is used from one host thread at a time (thread-compatible).
 *
 * Each group cites the reference interface it replaces (paths relative to
 * /root/reference/pearl, commit 48f1fbb).
 */
#ifndef PEARL_B200_H
#define PEARL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PRL_OK 0
#define PRL_EINVAL (-1)    /* contract violation (reference raises ValueError / assert) */
#define PRL_ECUDA (-2)     /* CUDA runtime error */
#define PRL_ENOMEM (-3)
#define PRL_ESTATE (-4)    /* call not valid in the handle's current state */
#define PRL_EUNSUPPORTED (-5)

#define PRL_ABI_VERSION 1

/* ---- library ----------------------------------------------------------- */
int prl_abi_version(void);
/* Select `device` for the calling thread and check it is sm_90 (H100).
 * There is no CPU fallback: without an H100 this returns PRL_EUNSUPPORTED. */
int prl_init(int device);
const char *prl_last_error(void);
/* multiprocessor count of the current device (grid sizing, reported by bench) */
int prl_sm_count(void);

/* ---- replay buffer ------------------------------------------------------
 * Replaces BasicReplayBuffer / TensorBasedReplayBuffer
 * (replay_buffers/basic_replay_buffer.py:17-48,
 *  replay_buffers/tensor_based_replay_buffer.py:55-133,253-288).
 *
 * Storage is ONE caller-allocated device array of `capacity` fixed-size
 * records ("array of transitions": sampling touches whole random transitions,
 * so a transition is contiguous, 16-byte aligned, and moves with one bulk
 * copy).  Record layout in 32-bit words (see prl_buf_layout):
 *     [off_state      .. +obs_dim)   state        f32
 *     [off_next_state .. +obs_dim)   next_state   f32
 *     [off_action     .. +act_words) action       i32 (discrete) | f32[act_dim]
 *     [off_reward]                   reward       f32
 *     [off_flags]                    bit0 terminated, bit1 truncated,
 *                                    bits 8..23 number of next available actions,
 *                                    bits 24..31 (PRL_BUF_NEXT_ACTION only) the
 *                                    committed next action id (SARSA)
 *     [off_avail .. ) (PRL_BUF_DYNAMIC_ACTIONS only) n_actions u8 ids of the
 *                     next available actions (padded with 0), as the reference
 *                     pads `next_available_actions` (tensor_based_replay_buffer.py:179-251)
 *     [cost]          (PRL_BUF_COST only) the transition's cost, f32, right after
 *                     everything above (prl_buf_cost_offset): no other offset moves
 * FIFO eviction like deque(maxlen=capacity): logical index 0 = oldest.
 */
#define PRL_BUF_DISCRETE 0x1          /* action is one int32 id in [0, n_actions) */
#define PRL_BUF_CONTINUOUS 0x2        /* action is act_dim floats */
#define PRL_BUF_DYNAMIC_ACTIONS 0x4   /* per-transition next-available-action sets */
#define PRL_BUF_NEXT_ACTION 0x8       /* discrete only: the committed next action id of SARSA in the flags word */
#define PRL_BUF_COST 0x10             /* one f32 cost per transition (TransitionBatch.cost, the reward-constrained safety module) */

typedef struct prl_buf_desc {
    int64_t capacity;
    int32_t obs_dim;
    int32_t act_dim;     /* continuous: action dimension; discrete: 1 */
    int32_t n_actions;   /* discrete: max_number_actions; continuous: 0 */
    int32_t flags;       /* PRL_BUF_* */
} prl_buf_desc;

typedef struct prl_buf_layout {
    int32_t record_words;   /* record stride in 32-bit words (multiple of 4) */
    int32_t off_state, off_next_state, off_action, off_reward, off_flags, off_avail;
    int32_t act_words;
    int64_t storage_bytes;  /* capacity * record_words * 4 */
} prl_buf_layout;

typedef struct prl_buf prl_buf;

int prl_buf_layout_of(const prl_buf_desc *desc, prl_buf_layout *out);
/* `storage_dev`: device memory of layout.storage_bytes bytes, 16-byte aligned.
 * `mt_state_dev`: device uint32[625], the MT19937 state in the layout of
 * CPython's random.getstate()[1] (624 words + position). */
int prl_buf_create(prl_buf **out, const prl_buf_desc *desc, void *storage_dev,
                   uint32_t *mt_state_dev);
int prl_buf_destroy(prl_buf *buf);
int64_t prl_buf_len(const prl_buf *buf);          /* __len__  (:284-285) */
int64_t prl_buf_capacity(const prl_buf *buf);
int64_t prl_buf_head(const prl_buf *buf);         /* physical slot of logical index 0 */
int prl_buf_clear(prl_buf *buf);                  /* clear()  (:287-288) */
/* Restore occupancy after the caller refilled `storage_dev` itself
 * (checkpoint load): `len` valid records, oldest at physical slot `head`. */
int prl_buf_set_occupancy(prl_buf *buf, int64_t len, int64_t head);

/* Multi-GPU: `buf` is rank `rank`'s shard of ONE logical replay buffer of `world * capacity` transitions
 * (SURVEY.md 8e; the reference has no sharded buffer — its BasicReplayBuffer is the world == 1 case,
 * basic_replay_buffer.py:21-48).  The transition with global write counter g lives on rank g mod world at
 * local slot (g div world) mod capacity, so FIFO eviction and age-uniform sampling stay balanced.
 * `global_pushed` = pushes to the logical buffer so far; the shard must hold exactly its share.  A sharded
 * buffer samples from the LOGICAL population: every rank runs the same MT19937 stream and draws the same
 * `batch` global indices as one GPU would (random.sample over the whole deque,
 * tensor_based_replay_buffer.py:276); prl_dqn_learn then works on the rows the rank owns. */
int prl_buf_set_shard(prl_buf *buf, int rank, int world, int64_t global_pushed);
int64_t prl_buf_global_len(const prl_buf *buf);

/* The same host push for `count` buffers of one record layout in ONE call (a vectorised environment feeding
 * a learner group): every source is a [count][n][...] host array; no per-transition action sets.  Records
 * are packed by a few worker threads and copied with one cudaMemcpyAsync per buffer. */
int prl_buf_push_host_multi(prl_buf *const *bufs, int count, int64_t n, const float *state, const void *action,
                            const float *reward, const float *next_state, const uint8_t *terminated,
                            const uint8_t *truncated, void *stream);

/* push n transitions given as HOST arrays (struct-of-arrays, C order):
 * state/next_state f32[n][obs_dim]; action int32[n] or f32[n][act_dim];
 * reward f32[n]; terminated/truncated u8[n]; next_avail_ids u8[n][n_actions]
 * and next_avail_cnt i32[n] (both NULL => all n_actions available).
 * Records are packed into the handle's pinned staging area and copied with
 * at most two cudaMemcpyAsync (ring wrap).  Replaces push() (:55-133) +
 * _store_transition (basic_replay_buffer.py:21-48), batched. */
int prl_buf_push_host(prl_buf *buf, int64_t n, const float *state, const void *action,
                      const float *reward, const float *next_state, const uint8_t *terminated,
                      const uint8_t *truncated, const uint8_t *next_avail_ids,
                      const int32_t *next_avail_cnt, void *stream);
/* same, sources already on the device (pack kernel, no host round trip) */
int prl_buf_push_device(prl_buf *buf, int64_t n, const float *state, const void *action,
                        const float *reward, const float *next_state, const uint8_t *terminated,
                        const uint8_t *truncated, const uint8_t *next_avail_ids,
                        const int32_t *next_avail_cnt, void *stream);

/* The pushes of a PRL_BUF_NEXT_ACTION buffer (SARSAReplayBuffer's complete tuples,
 * replay_buffers/sequential_decision_making/sarsa_replay_buffer.py:29-101): the
 * arguments of prl_buf_push_host / prl_buf_push_device / prl_buf_push_host_multi
 * plus next_action int32[n] (multi: [count][n]), ids in [0, n_actions) (host
 * pushes check them).  A PRL_BUF_NEXT_ACTION buffer refuses the plain entries, a
 * plain buffer refuses these (PRL_EINVAL): no next action is ever stored as id 0
 * by omission. */
int prl_buf_push_host_sarsa(prl_buf *buf, int64_t n, const float *state, const void *action,
                            const float *reward, const float *next_state, const uint8_t *terminated,
                            const uint8_t *truncated, const uint8_t *next_avail_ids,
                            const int32_t *next_avail_cnt, const int32_t *next_action, void *stream);
int prl_buf_push_device_sarsa(prl_buf *buf, int64_t n, const float *state, const void *action,
                              const float *reward, const float *next_state, const uint8_t *terminated,
                              const uint8_t *truncated, const uint8_t *next_avail_ids,
                              const int32_t *next_avail_cnt, const int32_t *next_action, void *stream);
int prl_buf_push_host_multi_sarsa(prl_buf *const *bufs, int count, int64_t n, const float *state,
                                  const void *action, const float *reward, const float *next_state,
                                  const uint8_t *terminated, const uint8_t *truncated,
                                  const int32_t *next_action, void *stream);

/* RNG state hand-off with CPython's global `random` module
 * (the reference samples with random.sample, tensor_based_replay_buffer.py:276;
 * state = random.getstate()[1]).  Host pointers, uint32[625].  get synchronises
 * `stream`. */
int prl_rng_set_state(prl_buf *buf, const uint32_t *state625_host, void *stream);
int prl_rng_get_state(prl_buf *buf, uint32_t *state625_host, void *stream);
/* random.seed(int): abs(seed) as little-endian 32-bit key words */
int prl_rng_seed(prl_buf *buf, const uint32_t *key_host, int key_len, void *stream);

/* Draw `rounds` consecutive samples of `k` distinct logical indices, exactly
 * the values `random.sample(range(len), k)` would return `rounds` times in a
 * row from the current MT19937 state (both CPython branches), advancing the
 * state.  out_logical_dev / out_slot_dev: device int32[rounds][k] (either may
 * be NULL); slot = physical record index.  PRL_EINVAL if k > len
 * (reference: ValueError, :271-275). */
int prl_buf_sample_indices(prl_buf *buf, int rounds, int k, int32_t *out_logical_dev,
                           int32_t *out_slot_dev, void *stream);

/* Gather k records into the reference's TransitionBatch field layout
 * (_create_transition_batch :290-400; dtypes of SURVEY.md §8 a4), all device
 * pointers, any of them may be NULL:
 *   state/next_state f32[k][obs_dim]; action i64[k] (discrete) or
 *   f32[k][act_dim]; reward f32[k]; terminated/truncated u8[k] (bool);
 *   next_avail f32[k][n_actions] (action ids, 0-padded);
 *   next_unavail_mask u8[k][n_actions] (1 = unavailable). */
int prl_buf_gather(const prl_buf *buf, const int32_t *slot_dev, int k, float *state, void *action,
                   float *reward, float *next_state, uint8_t *terminated, uint8_t *truncated,
                   float *next_avail, uint8_t *next_unavail_mask, void *stream);

/* The committed next action of k records of a PRL_BUF_NEXT_ACTION buffer:
 * out_dev i64[k] (the reference collates next_action as int64); PRL_EINVAL on
 * any other buffer. */
int prl_buf_gather_next_action(const prl_buf *buf, const int32_t *slot_dev, int k, int64_t *out_dev,
                               void *stream);

/* Costs (PRL_BUF_COST; the reference stores `cost` when the first pushed transition
 * has one, tensor_based_replay_buffer.py:55-133, and collates it into
 * TransitionBatch.cost).  The cost word follows every other field of the record, so
 * every offset of prl_buf_layout is the one the same flags without PRL_BUF_COST give.
 * prl_buf_cost_offset: *out = the cost word's offset in the record; PRL_EINVAL for a
 * descriptor without PRL_BUF_COST.
 * The pushes take the arguments of prl_buf_push_host / prl_buf_push_device plus
 * cost f32[n].  A PRL_BUF_COST buffer refuses the plain pushes (and the SARSA and
 * multi-buffer pushes), a plain buffer refuses these (PRL_EINVAL): no cost is ever
 * stored as 0 by omission.  A sharded PRL_BUF_COST buffer is refused by
 * prl_buf_set_shard.  prl_buf_gather_cost: out_dev f32[k]. */
int prl_buf_cost_offset(const prl_buf_desc *desc, int32_t *out);
int prl_buf_push_host_cost(prl_buf *buf, int64_t n, const float *state, const void *action,
                           const float *reward, const float *next_state, const uint8_t *terminated,
                           const uint8_t *truncated, const uint8_t *next_avail_ids,
                           const int32_t *next_avail_cnt, const float *cost, void *stream);
int prl_buf_push_device_cost(prl_buf *buf, int64_t n, const float *state, const void *action,
                             const float *reward, const float *next_state, const uint8_t *terminated,
                             const uint8_t *truncated, const uint8_t *next_avail_ids,
                             const int32_t *next_avail_cnt, const float *cost, void *stream);
int prl_buf_gather_cost(const prl_buf *buf, const int32_t *slot_dev, int k, float *out_dev, void *stream);

/* ---- DQN / DoubleDQN learner ---------------------------------------------
 * Replaces DeepTDLearning.learn_batch + DeepQLearning / DoubleDQN
 * .get_next_state_values + VanillaQValueNetwork.get_q_values + AdamW(amsgrad)
 * + update_target_network, driven by PolicyLearner.learn's training_rounds
 * loop (policy_learners/policy_learner.py:162-195,
 * policy_learners/sequential_decision_making/deep_td_learning.py:269-360,
 * deep_q_learning.py:130-167, double_dqn.py:29-57,
 * neural_networks/sequential_decision_making/q_value_networks.py:152-174,
 * neural_networks/common/utils.py:214-226, torch/optim/adam.py).
 *
 * Network: VanillaQValueNetwork with two hidden layers,
 *   x = [state | one_hot(action)]  ->  Linear(H1) ReLU Linear(H2) ReLU Linear(1).
 * Parameters are ONE flat fp32 array in torch's own parameter order and
 * layout (nn.Linear weight [out][in] row-major, then bias):
 *   W1[H1][obs+A] b1[H1] W2[H2][H1] b2[H2] W3[1][H2] b3[1]
 * so the caller can expose views of it as the module's state_dict.
 */
typedef struct prl_dqn_cfg {
    int32_t obs_dim, n_actions, hidden1, hidden2;
    int32_t double_dqn;            /* 0: DeepQLearning, 1: DoubleDQN */
    int32_t target_update_freq;    /* soft update when (training_steps+1) % freq == 0 */
    int32_t max_batch;             /* largest batch learn()/learn_batch() will be given */
    int32_t max_rounds;            /* largest `rounds` per prl_dqn_learn call */
    int32_t rows_per_cta;          /* 0 = choose automatically */
    /* AdamW (amsgrad always on), discount, soft-update coefficient: doubles,
     * because the reference evaluates these scalars in Python floats */
    double lr, beta1, beta2, eps, weight_decay;
    double gamma, tau;
} prl_dqn_cfg;

typedef struct prl_dqn prl_dqn;

int64_t prl_dqn_param_count(const prl_dqn_cfg *cfg);
/* bytes of device workspace the caller must provide to prl_dqn_create */
int64_t prl_dqn_workspace_bytes(const prl_dqn_cfg *cfg);
/* w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq: device f32[param_count].
 * adam_step: number of optimizer steps already taken (torch's `step`). */
int prl_dqn_create(prl_dqn **out, const prl_dqn_cfg *cfg, float *w, float *w_target,
                   float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq, int64_t adam_step,
                   void *workspace_dev);
int prl_dqn_destroy(prl_dqn *dqn);
int64_t prl_dqn_adam_step(const prl_dqn *dqn);
int prl_dqn_set_adam_step(prl_dqn *dqn, int64_t step);
int prl_dqn_set_lr(prl_dqn *dqn, double lr);

/* PolicyLearner.learn(replay_buffer) for `rounds` training rounds in ONE call:
 * draws rounds x batch indices (bit-exact with random.sample), then runs a
 * persistent kernel that per round gathers the batch, applies the scheduled
 * soft target update, computes Q(s,a), the Bellman target, the MSE gradient,
 * and the AdamW(amsgrad) step.  `training_steps0` is the learner's
 * `_training_steps` BEFORE the call (round r uses training_steps0 + r + 1).
 * out_mae_dev: device f32[rounds], the reference's reported "loss"
 * (mean |q - y|, deep_td_learning.py:358-360).  Optional device outputs for
 * parity tests (NULL to skip): out_q / out_y f32[rounds][batch],
 * out_logical i32[rounds][batch].  Asynchronous on `stream`. */
int prl_dqn_learn(prl_dqn *dqn, prl_buf *buf, int rounds, int batch, int64_t training_steps0,
                  float *out_mae_dev, float *out_q_dev, float *out_y_dev,
                  int32_t *out_logical_dev, void *stream);

/* DeepTDLearning.learn_batch(batch) on a caller-supplied TransitionBatch
 * (PearlAgent.learn_batch / offline learning, pearl_agent.py:222-231): device
 * arrays in prl_buf_gather's output layout; next_avail / mask may be NULL
 * (all actions available).  `do_target_update` = the caller's evaluation of
 * (training_steps+1) % freq == 0.  out_mae_dev: f32[1]. */
int prl_dqn_learn_batch(prl_dqn *dqn, int batch, const float *state, const int64_t *action,
                        const float *reward, const float *next_state, const uint8_t *terminated,
                        const float *next_avail, const uint8_t *next_unavail_mask,
                        int do_target_update, float *out_mae_dev, float *out_q_dev,
                        float *out_y_dev, void *stream);

/* Q(s, a) for every action (act(): deep_td_learning.py:200-254): device
 * state f32[n][obs_dim] -> out_q f32[n][n_actions], online (target=0) or
 * target network. */
int prl_dqn_q_values(prl_dqn *dqn, int n, const float *state, int target, float *out_q_dev,
                     void *stream);

/* how the last prl_dqn_learn was executed (bench / tests): number of kernel
 * launches, CTAs of the persistent learner kernel, rows per CTA */
int prl_dqn_last_launch_info(const prl_dqn *dqn, int32_t *launches, int32_t *ctas,
                             int32_t *rows_per_cta);

/* ---- multi-GPU data-parallel learner -------------------------------------
 * One process per GPU (torch.distributed provides the rendezvous only).  Each rank owns a replay
 * shard and samples its own batch; inside the persistent learner kernel the per-rank gradient
 * (P floats) is exchanged between phase A and the AdamW step by ONE-SHOT PUSH over NVLink peer
 * memory: every rank stores (gradient value, round sequence number) as one 8-byte word into every
 * peer's inbox (double-buffered by round parity); the owner of parameter i polls the W sequence
 * numbers of element i, sums the W values in rank order and divides by W — one-way NVLink latency,
 * no fence / flag round trip, no host involvement.  All ranks therefore apply bit-identical updates
 * (the mean gradient of the W*B sampled transitions).  The reference has no counterpart: no RL
 * learner in Pearl is distributed (SURVEY.md §5, §8e); this is the "all-reduce on the gradient
 * only" of the north star, fused into the step kernel instead of a separate NCCL launch.
 *
 * The communicator's buffers are library-allocated (cudaMalloc) so that they can be shared with
 * CUDA IPC: exchange the 128-byte blob of prl_comm_local_handles between all ranks (any byte
 * all-gather), then prl_comm_open_peers with the W blobs in rank order. */
typedef struct prl_comm prl_comm;
#define PRL_COMM_HANDLE_BYTES 128
int prl_comm_create(prl_comm **out, int rank, int world, int64_t max_param_count);
int prl_comm_local_handles(prl_comm *comm, uint8_t out_blob[PRL_COMM_HANDLE_BYTES]);
int prl_comm_open_peers(prl_comm *comm, const uint8_t *blobs /* [world][PRL_COMM_HANDLE_BYTES] */);
int prl_comm_destroy(prl_comm *comm);
/* attach (or detach with NULL) a communicator to a learner; every rank must then call
 * prl_dqn_learn with the same `rounds` */
int prl_dqn_set_comm(prl_dqn *dqn, prl_comm *comm);

/* ---- tensor-core learner, one SM per learner (aggregate mode) -----------------------------
 * PolicyLearner.learn() for `count` INDEPENDENT learners (seeds / agents; the reference runs those
 * as separate OS processes, utils/scripts/benchmark.py:80-116) in one launch: CTA i trains learner
 * dqns[i] on buffer bufs[i] for `rounds` gradient steps with every dense contraction on wgmma
 * (3xTF32, fp32 accumulation in registers).  Same arithmetic contract and outputs as prl_dqn_learn, per
 * learner; out_mae (required) / out_q / out_y / out_logical are arrays of `count` device pointers
 * (the optional arrays and their entries may be NULL).  Shape class: hidden [64,64], obs % 8 == 0
 * and <= 128, n_actions in {1,2,4,8,16}, DeepQLearning (not DoubleDQN), batch 128 or 256, all
 * learners with one configuration and one record layout; otherwise PRL_EUNSUPPORTED (use
 * prl_dqn_learn).  prl_dqn_tc_supported answers that question for one learner. */
int prl_dqn_tc_supported(const prl_dqn *dqn, int batch);
int prl_dqn_learn_multi(prl_dqn *const *dqns, prl_buf *const *bufs, int count, int rounds, int batch,
                        const int64_t *training_steps0, float *const *out_mae_dev, float *const *out_q_dev,
                        float *const *out_y_dev, int32_t *const *out_logical_dev, void *stream);

/* ---- prioritized replay (sum tree) ----------------------------------------------------------
 * NOT in the reference (no prioritized replay exists in Pearl @ 48f1fbb, SURVEY.md §0.3): parity is
 * pinned against oracle/per_oracle.py, the restatement of proportional prioritization (Schaul et al.
 * 2016) that both sides implement with bit-identical fp32 trees.  Leaves are the physical ring slots
 * of a replay buffer of `capacity` records.  The caller provides two device arrays of
 * prl_per_tree_floats(capacity) floats (sum tree, min tree) and one device float (running maximum
 * priority); prl_per_create initialises them on `stream`. */
typedef struct prl_per_cfg {
    int64_t capacity;
    double alpha, beta, eps;   /* p = (|td| + eps)^alpha ; w = (p_min / p)^beta */
    uint64_t seed;             /* Philox4x32-10 key of the stratified draws */
} prl_per_cfg;
typedef struct prl_per prl_per;
int64_t prl_per_tree_floats(int64_t capacity);
int prl_per_create(prl_per **out, const prl_per_cfg *cfg, float *sum_tree_dev, float *min_tree_dev,
                   float *max_priority_dev, void *stream);
int prl_per_destroy(prl_per *per);
int prl_per_set_beta(prl_per *per, double beta);
int64_t prl_per_draws(const prl_per *per);
/* transitions just written to ring slots [first_slot, first_slot + count) (wrapping) enter at the
 * running maximum priority */
int prl_per_push(prl_per *per, int64_t first_slot, int64_t count, void *stream);
/* k <= 1024 stratified draws: out_slots_dev i32[k] (ring slots), out_weights_dev f32[k] (IS weights) */
int prl_per_sample(prl_per *per, int k, int32_t *out_slots_dev, float *out_weights_dev, void *stream);
/* new priorities (|td| + eps)^alpha for k <= 1024 sampled slots; out_priority_dev (optional) f32[k] */
int prl_per_set_priorities(prl_per *per, const int32_t *slots_dev, const float *td_dev, int k,
                           float *out_priority_dev, void *stream);
/* PolicyLearner.learn() over a prioritized buffer: per round sample -> weighted MSE step (the IS weight
 * multiplies the squared TD error) -> priority update from |q - y|.  Same outputs as prl_dqn_learn;
 * out_slots_dev (optional) i32[rounds][batch] receives the sampled ring slots. */
int prl_dqn_learn_per(prl_dqn *dqn, prl_buf *buf, prl_per *per, int rounds, int batch, int64_t training_steps0,
                      float *out_mae_dev, float *out_q_dev, float *out_y_dev, int32_t *out_slots_dev,
                      float *out_weights_dev, void *stream);

/* ---- PPO preprocessing: GAE + truncated lambda returns --------------------------------------
 * Replaces the per-transition loop of ProximalPolicyOptimization.preprocess_replay_buffer
 * (policy_learners/sequential_decision_making/ppo.py:271-293).  All arrays are device pointers in
 * TIME order (index 0 = oldest stored transition): values[i] = critic(state_i), last_next_value =
 * critic(next_state of the newest transition), reward f32, terminated / truncated u8.  Outputs gae[i],
 * lam_return[i] are bit-identical to the reference loop (same fp32 operation order); episodes
 * (chains between terminated / truncated transitions) are processed in parallel.  scratch_dev: device int32[n + 1]
 * owned by the caller (the compacted chain heads and their count; contents are overwritten). */
int prl_ppo_gae(int n, const float *values_dev, float last_next_value, const float *reward_dev,
                const uint8_t *terminated_dev, const uint8_t *truncated_dev, double gamma, double lam,
                float *out_gae_dev, float *out_lam_return_dev, int32_t *scratch_dev, void *stream);

/* ---- continuous Soft Actor-Critic ---------------------------------------------------------------
 * Replaces ContinuousSoftActorCritic.learn_batch (policy_learners/sequential_decision_making/
 * actor_critic_base.py:309-366, soft_actor_critic_continuous.py:131-231) driven by PolicyLearner.learn
 * (policy_learner.py:162-204) over a continuous-action ring: per round sample -> actor step
 * (GaussianActorNetwork.sample_action, actor_networks.py:551-591, twin-critic minimum) -> critic step
 * with the updated actor (twin MSE against the entropy-regularised target, critic_utils.py:170-203)
 * -> soft target update (tau every step) -> entropy-coefficient step.  Three AdamW(amsgrad) states.
 * Flat parameter layouts (fp32, row-major [out][in] like nn.Linear):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 Wmu[A][h2] bmu Wstd[A][h2] bstd
 *   critic: TWO consecutive copies (q1 then q2) of W1[c1][obs+A] b1 W2[c2][c1] b2 W3[1][c2] b3
 * The reparameterisation noise is an input (device f32[rounds][2][batch][A]: first draw on `state`
 * for the actor loss, second on `next_state` for the target), as torch's Normal.rsample consumes it. */
typedef struct prl_sac_cfg {
    int32_t obs_dim, act_dim, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t autotune;     /* entropy_autotune */
    int32_t max_batch, max_rounds;
    double actor_lr, critic_lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_sac_cfg;
typedef struct prl_sac prl_sac;
int64_t prl_sac_actor_param_count(const prl_sac_cfg *cfg);
int64_t prl_sac_critic_param_count(const prl_sac_cfg *cfg);   /* ONE critic */
int64_t prl_sac_workspace_bytes(const prl_sac_cfg *cfg);
/* All pointers are device memory owned by the caller: actor vectors f32[actor_param_count], critic
 * vectors f32[2 * critic_param_count], log_alpha4 = {log_alpha, exp_avg, exp_avg_sq, max_exp_avg_sq},
 * alpha1 = the entropy coefficient in use, low/high f32[act_dim] action-space bounds. */
int prl_sac_create(prl_sac **out, const prl_sac_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                   float *actor_vmax, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                   float *critic_target_w, float *log_alpha4, float *alpha1, const float *low_dev,
                   const float *high_dev, int64_t adam_step, void *workspace);
int prl_sac_destroy(prl_sac *sac);
int64_t prl_sac_adam_step(const prl_sac *sac);
/* out_*_loss: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices */
int prl_sac_learn(prl_sac *sac, prl_buf *buf, int rounds, int batch, const float *noise_dev,
                  float *out_actor_loss_dev, float *out_critic_loss_dev, float *out_entropy_loss_dev,
                  int32_t *out_logical_dev, void *stream);
/* The round is a fixed sequence of kernel launches replayed from a CUDA graph (default on; 0 = plain
 * stream launches, e.g. under a profiler).  prl_sac_last_launches: kernels launched by the last learn. */
int prl_sac_set_graph(prl_sac *sac, int enable);
int64_t prl_sac_last_launches(const prl_sac *sac);

/* ---- discrete Soft Actor-Critic ----------------------------------------------------------------
 * Replaces SoftActorCritic.learn_batch (policy_learners/sequential_decision_making/soft_actor_critic.py:
 * learn_batch, _actor_loss, _critic_loss, _get_next_state_expected_values on actor_critic_base.py:309-366)
 * driven by PolicyLearner.learn (policy_learner.py:162-204) over a discrete-action ring: per round sample ->
 * actor step (VanillaActorNetwork softmax against min(Q1, Q2) of every action, the pre-step coefficient) ->
 * critic step with the updated actor and the critic target (twin MSE, critic_utils.py) -> soft target update
 * (tau every round) -> entropy step (torch.optim.Adam on log alpha, with the actor-step probabilities).
 * Two AdamW(amsgrad) states (actor, both critics).  Flat layouts (fp32, row-major [out][in]):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 W3[A][h2] b3
 *   critic: TWO consecutive copies (q1 then q2) of W1[c1][obs+A] b1 W2[c2][c1] b2 W3[1][c2] b3 (one-hot action)
 * target_entropy = -scale * log(1 / A) as the reference computes it; entropy_lr / entropy_eps are the entropy
 * optimizer's (the critic lr at construction, 1e-4).  Sharded and continuous-action buffers are rejected (EINVAL). */
typedef struct prl_sacd_cfg {
    int32_t obs_dim, n_actions, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t autotune;     /* entropy_autotune */
    int32_t max_batch, max_rounds;
    double actor_lr, critic_lr, beta1, beta2, eps, weight_decay, gamma, tau;
    double target_entropy, entropy_lr, entropy_eps;
} prl_sacd_cfg;
typedef struct prl_sacd prl_sacd;
int64_t prl_sacd_actor_param_count(const prl_sacd_cfg *cfg);
int64_t prl_sacd_critic_param_count(const prl_sacd_cfg *cfg);   /* ONE critic */
int64_t prl_sacd_workspace_bytes(const prl_sacd_cfg *cfg);
/* Device memory owned by the caller: actor vectors f32[actor_param_count], critic vectors f32[2 * critic_param_count],
 * log_alpha3 = {log_alpha, exp_avg, exp_avg_sq} (torch.optim.Adam state), alpha1 = the entropy coefficient in use. */
int prl_sacd_create(prl_sacd **out, const prl_sacd_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                    float *actor_vmax, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                    float *critic_target_w, float *log_alpha3, float *alpha1, int64_t adam_step, void *workspace);
int prl_sacd_destroy(prl_sacd *sacd);
int64_t prl_sacd_adam_step(const prl_sacd *sacd);
/* New actor / critic AdamW learning rates from the next learn on (an lr scheduler's step, e.g. the ExponentialLR
 * that SoftActorCritic.reset steps).  Every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_sacd_set_lr(prl_sacd *sacd, double actor_lr, double critic_lr);
/* out_*_loss: device f32[rounds] (entropy: the entropy optimizer's loss, as the reference reports it);
 * out_logical_dev (optional) i32[rounds][batch] = sampled indices */
int prl_sacd_learn(prl_sacd *sacd, prl_buf *buf, int rounds, int batch, float *out_actor_loss_dev,
                   float *out_critic_loss_dev, float *out_entropy_loss_dev, int32_t *out_logical_dev, void *stream);
int prl_sacd_set_graph(prl_sacd *sacd, int enable);
int64_t prl_sacd_last_launches(const prl_sacd *sacd);

/* ---- TD3 / DDPG ----------------------------------------------------------------------------------
 * Replaces TD3.learn_batch (policy_learners/sequential_decision_making/td3.py:106-202) and, with
 * actor_update_freq = 1 and no noise, DeepDeterministicPolicyGradient (ddpg.py:105-157 on
 * actor_critic_base.py:309-366), driven by PolicyLearner.learn (policy_learner.py:162-204) over a
 * continuous-action ring: per round sample -> [if training_steps % actor_update_freq == 0: actor step,
 * maximise Q1(s, pi(s)), VanillaContinuousActorNetwork tanh head + action_scaling, actor_networks.py:29-51,448-485]
 * -> twin-critic step against min(Q1', Q2')(s', clamp(pi'(s') + clipped noise)) -> [on the same rounds: soft
 * update of the critic targets and of the actor target].  The actor optimizer's step count advances only on its
 * update rounds.  Flat layouts (fp32, row-major [out][in]):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 W3[A][h2] b3       critic: as prl_sac (q1 then q2)
 * noise_dev: device f32[rounds][batch][A] = the torch.normal(0, actor_update_noise, ...) draws (null: DDPG). */
typedef struct prl_td3_cfg {
    int32_t obs_dim, act_dim, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t actor_update_freq;
    int32_t max_batch, max_rounds;
    double actor_lr, critic_lr, beta1, beta2, eps, weight_decay, gamma, actor_tau, critic_tau, noise_clip;
} prl_td3_cfg;
typedef struct prl_td3 prl_td3;
int64_t prl_td3_actor_param_count(const prl_td3_cfg *cfg);
int64_t prl_td3_critic_param_count(const prl_td3_cfg *cfg);   /* ONE critic */
int64_t prl_td3_workspace_bytes(const prl_td3_cfg *cfg);
int prl_td3_create(prl_td3 **out, const prl_td3_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                   float *actor_vmax, float *actor_target_w, float *critic_w, float *critic_m, float *critic_v,
                   float *critic_vmax, float *critic_target_w, const float *low_dev, const float *high_dev,
                   int64_t actor_adam_step, int64_t critic_adam_step, void *workspace);
int prl_td3_destroy(prl_td3 *td3);
int64_t prl_td3_actor_adam_step(const prl_td3 *td3);
int64_t prl_td3_critic_adam_step(const prl_td3 *td3);
/* training_steps0 = learner._training_steps before the call; out_*_loss: device f32[rounds] */
int prl_td3_learn(prl_td3 *td3, prl_buf *buf, int rounds, int batch, int64_t training_steps0, const float *noise_dev,
                  float *out_actor_loss_dev, float *out_critic_loss_dev, int32_t *out_logical_dev, void *stream);
int prl_td3_set_graph(prl_td3 *td3, int enable);
int64_t prl_td3_last_launches(const prl_td3 *td3);
/* Rounds captured as CUDA graphs so far.  Ring and dense-batch rounds, with and without the actor update, are kept
 * side by side: alternating learn and learn_batch captures nothing after the first of each. */
int64_t prl_td3_graph_captures(const prl_td3 *td3);
/* One round on the caller's dense batch: TD3.learn_batch (td3.py:106-147) / ActorCriticBase.learn_batch
 * (actor_critic_base.py:309-366), as PearlAgent.learn_batch and offline_learning() call it
 * (offline_learning_and_evaluation.py:217-224).  training_steps = learner._training_steps as it is (learn_batch does not
 * advance it): the actor and target updates run when training_steps % actor_update_freq == 0.
 * state / next_state: device f32[batch][obs]; action: f32[batch][A]; reward: f32[batch]; terminated: u8[batch];
 * noise_dev: f32[1][batch][A] (null: DDPG); out_*_loss: device f32[1]. */
int prl_td3_learn_batch(prl_td3 *td3, int batch, const float *state, const float *action, const float *reward,
                        const float *next_state, const uint8_t *terminated, int64_t training_steps, const float *noise_dev,
                        float *out_actor_loss_dev, float *out_critic_loss_dev, void *stream);
/* The loss a round without an actor update reports: TD3's _last_actor_loss (td3.py:104,122).  A handle starts at 0; a
 * handle re-created mid-training (a learning-rate change, a larger batch) is seeded with the learner's value. */
int prl_td3_set_last_actor_loss(prl_td3 *td3, float value);

/* ---- TD3BC (offline TD3 with a behaviour-cloning actor term) -------------------------------------
 * Replaces TD3BC._actor_loss (policy_learners/sequential_decision_making/td3.py:298-318) inside the TD3 round above:
 *   a = sample_action(s) (tanh, scaled to the box), q = Q1(s, a), b = behavior_policy(s) under no_grad,
 *   lambda = alpha_bc / mean|q| (detached), loss = mean((a - b)^2) - lambda mean(q).
 * behavior_policy is a VanillaContinuousActorNetwork called through forward(): b is the raw tanh output in [-1, 1], not
 * scaled to the box (actor_networks.py:472-473).  Behaviour weights: device f32, flat W1[h1][obs] b1 W2[h2][h1] b2
 * W3[A][h2] b3, read by every round (not copied).  The handle is a prl_td3: destroy, step counts, set_graph, learn,
 * learn_batch and the setters above apply to it. */
typedef struct prl_td3bc_cfg {
    int32_t behavior_h1, behavior_h2;
} prl_td3bc_cfg;
int64_t prl_td3bc_workspace_bytes(const prl_td3_cfg *cfg, const prl_td3bc_cfg *bc);
int prl_td3bc_create(prl_td3 **out, const prl_td3_cfg *cfg, const prl_td3bc_cfg *bc, const float *behavior_w, float *actor_w,
                     float *actor_m, float *actor_v, float *actor_vmax, float *actor_target_w, float *critic_w,
                     float *critic_m, float *critic_v, float *critic_vmax, float *critic_target_w, const float *low_dev,
                     const float *high_dev, int64_t actor_adam_step, int64_t critic_adam_step, void *workspace);
/* TD3BC.alpha_bc (td3.py:295), read by the next call; TD3BC handles only */
int prl_td3_set_alpha_bc(prl_td3 *td3, double alpha_bc);

/* Cost-shaped rewards (ActorCriticBase.preprocess_batch, actor_critic_base.py:368-383, with a reward-constrained safety
 * module): enable != 0 makes every round of the next prl_td3_learn calls train on reward - fp32(lambda) * cost, two
 * rounded fp32 operations as torch evaluates them, with the cost read from the ring (a PRL_BUF_COST buffer: prl_td3_learn
 * refuses any other while shaping is on).  lambda travels in the per-call block: changing it never re-captures a round.
 * prl_td3_learn_batch never shapes (its batch is already preprocessed).  A handle starts with shaping off. */
int prl_td3_set_cost_lambda(prl_td3 *td3, int enable, double lambda);

/* ---- reward-constrained safety module (the cost critic and the Lagrange multiplier) ----------------
 * Replaces RCSafetyModuleCostCriticContinuousAction.learn (safety_modules/reward_constrained_safety_module.py:115-216)
 * for a TD3 / DDPG / TD3BC policy learner, called once per PearlAgent.learn after the policy learner's rounds
 * (pearl_agent.py:213-220).  One call = one sample of `batch` indices (continuing the buffer's MT19937 stream) and one
 * fixed launch sequence, captured as a CUDA graph:
 *   a' = actor(s') (VanillaContinuousActorNetwork.sample_action: tanh scaled to the box, no noise),
 *   y = min(Qc1', Qc2')(s', a') * cost_gamma * (1 - terminated) + cost,
 *   twin MSE loss (mse1 + mse2) / 2 (critic_utils.py:170-203), AdamW(amsgrad) step with the soft update of the target
 *   twin (every call), cq = mean(max(Qc1, Qc2)(s, actor(s))) with the UPDATED twin (one CTA, fixed order),
 *   lambda = clip(lambda + lr_lambda * (cq * (1 - cost_gamma) - constraint_value), 0, lambda_ub) in float64 with the
 *   reference's Python evaluation order.
 * The twin cost critic, its target and the AdamW vectors are caller-owned (flat as prl_sac's critic: q1 then q2).  The
 * policy's actor weights, its box and the multiplier travel in the per-call step block, so a re-created policy learner
 * needs no new handle.  The host never waits inside prl_rcsafety_learn. */
typedef struct prl_rcsafety_cfg {
    int32_t obs_dim, act_dim, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t max_batch;
    double critic_lr, beta1, beta2, eps, weight_decay, cost_gamma, tau;
} prl_rcsafety_cfg;
typedef struct prl_rcsafety_step {
    const float *actor_w;           /* device: the policy's actor, flat W1 b1 W2 b2 W3 b3 (prl_td3's layout) */
    const float *low, *high;        /* device f32[act_dim]: the box the actor scales to */
    double lambda_in, constraint_value, lr_lambda, lambda_ub;
    double *out;                    /* device f64[3]: the new lambda, the cost-critic loss, cq */
} prl_rcsafety_step;
typedef struct prl_rcsafety prl_rcsafety;
int64_t prl_rcsafety_param_count(const prl_rcsafety_cfg *cfg);   /* ONE cost critic; the twin vector holds two */
int64_t prl_rcsafety_workspace_bytes(const prl_rcsafety_cfg *cfg);
int prl_rcsafety_create(prl_rcsafety **out, const prl_rcsafety_cfg *cfg, float *critic_w, float *critic_m, float *critic_v,
                        float *critic_vmax, float *critic_target_w, int64_t adam_step, void *workspace);
int prl_rcsafety_destroy(prl_rcsafety *rc);
int64_t prl_rcsafety_adam_step(const prl_rcsafety *rc);
int prl_rcsafety_set_graph(prl_rcsafety *rc, int enable);
int64_t prl_rcsafety_graph_captures(const prl_rcsafety *rc);
int64_t prl_rcsafety_last_launches(const prl_rcsafety *rc);
/* buf: a local continuous-action PRL_BUF_COST buffer of the configured dimensions.  out_logical_dev: optional device
 * i32[batch], the sampled logical indices. */
int prl_rcsafety_learn(prl_rcsafety *rc, prl_buf *buf, int batch, const prl_rcsafety_step *step, int32_t *out_logical_dev,
                       void *stream);

/* ---- Implicit Q-Learning (offline actor-critic) ----------------------------------------------------
 * Replaces ImplicitQLearning.learn_batch (policy_learners/sequential_decision_making/implicit_q_learning.py:159-302),
 * driven by PolicyLearner.learn (prl_iql_learn: sample -> round, `rounds` times) or called on a caller's batch
 * (prl_iql_learn_batch: one round; offline_learning() drives the agent this way).  Per round, every loss from the
 * parameters before the round: value loss mean(w u^2), u = tq - V(s), w = expectile if u > 0 else 1 - expectile;
 * twin critic loss against r + gamma (1 - terminated) V(s') (critic_utils.py:170-203); advantage-weighted actor loss with
 * adv = min(exp((tq - V(s)) temperature), advantage_clamp); tq is q1 or q2 of the critic TARGET at (s, a), picked by the
 * round's two bits.  Then the value, critic and actor AdamW(amsgrad) steps (one shared step count) and the soft update of
 * the critic targets.  Discrete (n_actions > 0, act_dim = 0): VanillaActorNetwork, L = -mean(adv log softmax[a]), one-hot
 * critic input.  Continuous (act_dim > 0, n_actions = 0): VanillaContinuousActorNetwork (tanh scaled to [low, high]),
 * L = mean(adv mean_d (mu - a)^2).  Flat layouts (fp32, row-major [out][in]):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 W3[N][h2] b3        (N = n_actions or act_dim)
 *   critic: TWO consecutive copies (q1 then q2) of W1[c1][obs+N] b1 W2[c2][c1] b2 W3[1][c2] b3
 *   value : W1[v1][obs] b1 W2[v2][v1] b2 W3[1][v2] b3
 * bits_dev: device i32[rounds][2] = the round's torch.randint(0, 2) draws (value loss first, then actor loss).
 * Sharded buffers, buffers of the other action kind or other dimensions, and batch / rounds above the configured
 * maxima are rejected (EINVAL) before any launch. */
typedef struct prl_iql_cfg {
    int32_t obs_dim, n_actions, act_dim, actor_h1, actor_h2, critic_h1, critic_h2, value_h1, value_h2;
    int32_t max_batch, max_rounds;
    double actor_lr, critic_lr, value_lr, beta1, beta2, eps, weight_decay, gamma, tau;
    double expectile, temperature, advantage_clamp;
} prl_iql_cfg;
typedef struct prl_iql prl_iql;
int64_t prl_iql_actor_param_count(const prl_iql_cfg *cfg);
int64_t prl_iql_critic_param_count(const prl_iql_cfg *cfg);   /* ONE critic */
int64_t prl_iql_value_param_count(const prl_iql_cfg *cfg);
int64_t prl_iql_workspace_bytes(const prl_iql_cfg *cfg);
/* Device memory owned by the caller: actor vectors f32[actor_param_count], critic vectors f32[2 * critic_param_count],
 * value vectors f32[value_param_count]; low/high f32[act_dim] (continuous only, may be null when discrete). */
int prl_iql_create(prl_iql **out, const prl_iql_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                   float *actor_vmax, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                   float *critic_target_w, float *value_w, float *value_m, float *value_v, float *value_vmax,
                   const float *low_dev, const float *high_dev, int64_t adam_step, void *workspace);
int prl_iql_destroy(prl_iql *iql);
int64_t prl_iql_adam_step(const prl_iql *iql);
/* New AdamW learning rates from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_iql_set_lr(prl_iql *iql, double actor_lr, double critic_lr, double value_lr);
/* out_*_loss: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices */
int prl_iql_learn(prl_iql *iql, prl_buf *buf, int rounds, int batch, const int32_t *bits_dev, float *out_value_loss_dev,
                  float *out_critic_loss_dev, float *out_actor_loss_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action f32[batch][act_dim] (continuous) or
 * action_id i32[batch] (discrete), reward f32[batch], terminated u8[batch]; out_*_loss: device f32[1]. */
int prl_iql_learn_batch(prl_iql *iql, int batch, const float *state, const float *action, const int32_t *action_id,
                        const float *reward, const float *next_state, const uint8_t *terminated, const int32_t *bits_dev,
                        float *out_value_loss_dev, float *out_critic_loss_dev, float *out_actor_loss_dev, void *stream);
int prl_iql_set_graph(prl_iql *iql, int enable);
int64_t prl_iql_last_launches(const prl_iql *iql);

/* ---- Quantile Regression DQN -------------------------------------------------------------------------
 * Replaces QuantileRegressionDeepTDLearning.learn_batch (policy_learners/sequential_decision_making/
 * quantile_regression_deep_td_learning.py) with QuantileRegressionDeepQLearning._get_next_state_quantiles
 * (quantile_regression_deep_q_learning.py), the QuantileQValueNetwork (neural_networks/sequential_decision_making/
 * q_value_networks.py: mlp_block(state || one-hot(action)) -> N quantiles) and the risk metrics of
 * safety_modules/risk_sensitive_safety_modules.py, driven by PolicyLearner.learn (prl_qrdqn_learn: sample -> round,
 * `rounds` times) or called on a caller's batch (prl_qrdqn_learn_batch: one round).  Per round:
 *   theta_i(s, a) of the online net; theta'_j(s', k) of the target net for every next-action slot k;
 *   rho_k = mean_j theta'_j - beta sum_j w_j (theta'_j - mean)^2, w_j = (j+1)/N - j/N in fp32, -inf on masked slots;
 *   g = first argmax; T_j = theta'_j(s', g) gamma (1 - terminated) + r;
 *   L = mean over (b, i) of sum_j |tau^_i - 1{u < 0}| huber(u), u = T_j - theta_i, tau^_i = (i/N + (i+1)/N) / 2, kappa = 1;
 *   one AdamW(amsgrad) step; then, when (training_steps + 1) % target_update_freq == 0 with training_steps the count the
 *   reference's learn_batch sees, the soft update target = tau * online + (1 - tau) * target with the NEW parameters.
 *   Reported loss: mean over (b, i) of |theta_i - T_i|.
 * beta = 0 is RiskNeutralSafetyModule, beta > 0 QuantileNetworkMeanVarianceSafetyModule(beta).  1 <= num_quantiles <= 256,
 * 1 <= n_actions <= 255.  Flat layout (fp32, row-major [out][in]): W1[h1][obs + A] b1 W2[h2][h1] b2 W3[N][h2] b3.
 * Sharded buffers, continuous-action buffers, buffers of other obs_dim / n_actions, and batch / rounds above the
 * configured maxima are rejected (EINVAL) before any launch. */
typedef struct prl_qrdqn_cfg {
    int32_t obs_dim, n_actions, hidden1, hidden2, num_quantiles, target_update_freq;
    int32_t max_batch, max_rounds;
    double lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_qrdqn_cfg;
typedef struct prl_qrdqn prl_qrdqn;
int64_t prl_qrdqn_param_count(const prl_qrdqn_cfg *cfg);
int64_t prl_qrdqn_workspace_bytes(const prl_qrdqn_cfg *cfg);
/* Device memory owned by the caller: f32[param_count] each (online, target, AdamW exp_avg / exp_avg_sq / max_exp_avg_sq). */
int prl_qrdqn_create(prl_qrdqn **out, const prl_qrdqn_cfg *cfg, float *q_w, float *q_m, float *q_v, float *q_vmax,
                     float *q_target_w, int64_t adam_step, void *workspace);
int prl_qrdqn_destroy(prl_qrdqn *qr);
int64_t prl_qrdqn_adam_step(const prl_qrdqn *qr);
/* New AdamW learning rate from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_qrdqn_set_lr(prl_qrdqn *qr, double lr);
/* training_steps = the learner's count before the call (PolicyLearner.learn increments it before each round);
 * out_loss_dev: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices */
int prl_qrdqn_learn(prl_qrdqn *qr, prl_buf *buf, int rounds, int batch, int64_t training_steps, double beta,
                    float *out_loss_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action_id i32[batch], reward f32[batch],
 * terminated u8[batch], next_ids i32[batch][n_actions] (slot k holds an action id) and next_count i32[batch] (slots at
 * and beyond it are unavailable), both null when every action is available; training_steps = the count learn_batch sees
 * (agent.learn_batch does not advance it); out_loss_dev: device f32[1]. */
int prl_qrdqn_learn_batch(prl_qrdqn *qr, int batch, const float *state, const int32_t *action_id, const float *reward,
                          const float *next_state, const uint8_t *terminated, const int32_t *next_ids,
                          const int32_t *next_count, int64_t training_steps, double beta, float *out_loss_dev, void *stream);
int prl_qrdqn_set_graph(prl_qrdqn *qr, int enable);
int64_t prl_qrdqn_last_launches(const prl_qrdqn *qr);

/* ---- conservative DQN / DoubleDQN (CQL) ----------------------------------------------------------
 * Replaces DeepTDLearning.forward / loss / learn_batch with is_conservative=True (policy_learners/
 * sequential_decision_making/deep_td_learning.py:269-360), DeepQLearning / DoubleDQN.get_next_state_values
 * (deep_q_learning.py:130-167, double_dqn.py:29-57), compute_cql_loss (utils/functional_utils/learning/loss_fn_utils.py:
 * 17-71) and VanillaQValueNetwork.get_q_values (neural_networks/sequential_decision_making/q_value_networks.py:152-174),
 * driven by PolicyLearner.learn (prl_cql_learn: sample -> round, `rounds` times) or called on a caller's batch
 * (prl_cql_learn_batch: one round, PearlAgent.learn_batch / offline_learning).  Per round:
 *   when (training_steps + 1) % target_update_freq == 0, FIRST target = tau * online + (1 - tau) * target;
 *   q_b = Q(s_b, a_b); y_b = V_b gamma (1 - terminated_b) + r_b with V_b = max over available next slots of Q'(s'_b, .)
 *   (DQN) or Q'(s'_b, first argmax over available next slots of Q(s'_b, .)) (DoubleDQN);
 *   L = mean_b (q_b - y_b)^2 + alpha cql, cql = mean_b logsumexp_k Q(s_b, c_b[k]) - (1 / (B A)) sum_b [(A - 1) Q(s_b, c_b[0])
 *   + Q(s_b, c_b[1])]: the reference gathers the current-action values with the ONE-HOT action, so its second term reads
 *   columns 0 and 1, not the taken action; c_b[k] are the current slots including padding (id 0);
 *   one AdamW(amsgrad) step.  Reported loss: mean_b |q_b - y_b| (the Bellman error only).
 * 2 <= n_actions <= 255 (A = 1 makes the reference's gather index out of range); max_batch (n_actions + 1)
 * max(hidden1, hidden2) < 2^31 (32-bit element offsets of the slot rows; param_count / workspace_bytes return -1 and
 * create returns EINVAL beyond it).  Flat layout (fp32, row-major [out][in]):
 * W1[h1][obs + A] b1 W2[h2][h1] b2 W3[1][h2] b3, as prl_dqn.  Sharded buffers, continuous-action buffers, buffers of
 * other obs_dim / n_actions, and batch / rounds above the configured maxima are rejected (EINVAL) before any launch. */
typedef struct prl_cql_cfg {
    int32_t obs_dim, n_actions, hidden1, hidden2;
    int32_t double_dqn;            /* 0: DeepQLearning, 1: DoubleDQN */
    int32_t target_update_freq, max_batch, max_rounds;
    double lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_cql_cfg;
typedef struct prl_cql prl_cql;
int64_t prl_cql_param_count(const prl_cql_cfg *cfg);
int64_t prl_cql_workspace_bytes(const prl_cql_cfg *cfg);
/* w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq: device f32[param_count] owned by the caller (the argument order of
 * prl_dqn_create); adam_step: optimizer steps already taken (torch's `step`). */
int prl_cql_create(prl_cql **out, const prl_cql_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                   float *max_exp_avg_sq, int64_t adam_step, void *workspace_dev);
int prl_cql_destroy(prl_cql *cql);
int64_t prl_cql_adam_step(const prl_cql *cql);
int prl_cql_set_adam_step(prl_cql *cql, int64_t step);
/* New AdamW learning rate from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_cql_set_lr(prl_cql *cql, double lr);
/* training_steps = the learner's count before the call (PolicyLearner.learn increments it before each round); alpha =
 * conservative_alpha; out_loss_dev: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices.
 * The ring stores no current action sets: every round uses the full set, as B200ReplayBuffer.sample reports it. */
int prl_cql_learn(prl_cql *cql, prl_buf *buf, int rounds, int batch, int64_t training_steps, double alpha,
                  float *out_loss_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action_id i32[batch], reward f32[batch],
 * terminated u8[batch]; curr_ids i32[batch][n_actions] (slot k of the current set, padding included), null = every
 * action; next_ids i32[batch][n_actions] and next_count i32[batch] (slots at and beyond it are unavailable), both null
 * when every action is available next; training_steps = the count learn_batch sees (agent.learn_batch does not advance
 * it); out_loss_dev: device f32[1]. */
int prl_cql_learn_batch(prl_cql *cql, int batch, const float *state, const int32_t *action_id, const float *reward,
                        const float *next_state, const uint8_t *terminated, const int32_t *curr_ids, const int32_t *next_ids,
                        const int32_t *next_count, int64_t training_steps, double alpha, float *out_loss_dev, void *stream);
/* Q(s, a) for every action (DeepTDLearning.act, deep_td_learning.py:200-254): device state f32[n][obs_dim] ->
 * out_q f32[n][n_actions], online (target = 0) or target network. */
int prl_cql_q_values(prl_cql *cql, int n, const float *state, int target, float *out_q_dev, void *stream);
int prl_cql_set_graph(prl_cql *cql, int enable);
int64_t prl_cql_last_launches(const prl_cql *cql);

/* ---- dueling DQN / DoubleDQN --------------------------------------------------------------------
 * Replaces DuelingQValueNetwork.get_q_values (neural_networks/sequential_decision_making/q_value_networks.py:352-510),
 * DeepTDLearning.forward / loss / learn_batch (policy_learners/sequential_decision_making/deep_td_learning.py:269-360) and
 * DeepQLearning / DoubleDQN.get_next_state_values (deep_q_learning.py:130-167, double_dqn.py:29-57), driven by
 * PolicyLearner.learn (prl_duel_learn: sample -> round, `rounds` times) or called on a caller's batch (prl_duel_learn_batch:
 * one round, PearlAgent.learn_batch).  The network: state_arch obs -> state_h1 -> state_h2 -> feature_dim (no ReLU on the
 * feature), value_arch feature_dim -> value_h1 -> value_h2 -> 1, advantage_arch (feature || one-hot action) -> adv_h1 ->
 * adv_h2 -> 1; Q(s, a) = fl(fl(V(s) + Adv(s, a)) - mean of Adv(s, .) over a set that depends on the caller:
 *   online q: the A current slots, padding (id 0) included; the query action alone when learn_batch gets no current ids;
 *   DQN target: max over the available next slots, the mean over all A next slots (unavailable ones with their ids);
 *   DoubleDQN target: a* = first argmax over the available next slots of the online Q (mean over all A next slots), then
 *   V' = fl(fl(V_t(s') + Adv_t(s', a*)) - Adv_t(s', a*)) (the target net called with the single query a*).
 * Per round: when (training_steps + 1) % target_update_freq == 0, FIRST target = tau * online + (1 - tau) * target;
 * y = V' gamma (1 - terminated) + r; L = mean (q - y)^2; one AdamW(amsgrad) step.  Reported loss: mean |q - y|.
 * 1 <= n_actions <= 255; max_batch (n_actions + 1) max(adv_h1, adv_h2) < 2^31 (32-bit element offsets of the slot rows;
 * param_count / workspace_bytes return -1 and create returns EINVAL beyond it).  Flat layout (fp32, row-major [out][in],
 * torch's parameter order): state_arch W1 b1 W2 b2 W3 b3,
 * value_arch W1 b1 W2 b2 W3 b3, advantage_arch W1 b1 W2 b2 W3 b3.  Sharded buffers, continuous-action buffers, buffers of
 * other obs_dim / n_actions, and batch / rounds above the configured maxima are rejected (EINVAL) before any launch. */
typedef struct prl_duel_cfg {
    int32_t obs_dim, n_actions, feature_dim;   /* feature_dim: output width of state_arch (hidden_dims[-1]) */
    int32_t state_h1, state_h2, value_h1, value_h2, adv_h1, adv_h2;
    int32_t double_dqn;            /* 0: DeepQLearning, 1: DoubleDQN */
    int32_t target_update_freq, max_batch, max_rounds;
    double lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_duel_cfg;
typedef struct prl_duel prl_duel;
int64_t prl_duel_param_count(const prl_duel_cfg *cfg);
int64_t prl_duel_workspace_bytes(const prl_duel_cfg *cfg);
/* w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq: device f32[param_count] owned by the caller (the argument order of
 * prl_dqn_create); adam_step: optimizer steps already taken (torch's `step`). */
int prl_duel_create(prl_duel **out, const prl_duel_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                    float *max_exp_avg_sq, int64_t adam_step, void *workspace_dev);
int prl_duel_destroy(prl_duel *duel);
int64_t prl_duel_adam_step(const prl_duel *duel);
int prl_duel_set_adam_step(prl_duel *duel, int64_t step);
/* New AdamW learning rate from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_duel_set_lr(prl_duel *duel, double lr);
/* training_steps = the learner's count before the call (PolicyLearner.learn increments it before each round);
 * out_loss_dev: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices.  The ring stores no
 * current action sets: the online mean runs over every action, as B200ReplayBuffer.sample reports the set. */
int prl_duel_learn(prl_duel *duel, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss_dev,
                   int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action_id i32[batch], reward f32[batch],
 * terminated u8[batch]; curr_ids i32[batch][n_actions] (slot k of the current set, padding included), null = the online
 * mean runs over the query action alone; next_ids i32[batch][n_actions] (every slot, unavailable ones included: they
 * enter the mean with these ids), null = slot k holds k; next_unavailable u8[batch][n_actions] (1 = unavailable), null =
 * every slot available; training_steps = the count learn_batch sees (agent.learn_batch does not advance it);
 * out_loss_dev: device f32[1]. */
int prl_duel_learn_batch(prl_duel *duel, int batch, const float *state, const int32_t *action_id, const float *reward,
                         const float *next_state, const uint8_t *terminated, const int32_t *curr_ids, const int32_t *next_ids,
                         const uint8_t *next_unavailable, int64_t training_steps, float *out_loss_dev, void *stream);
/* Q(s, .) over an id set (DeepTDLearning.act, deep_td_learning.py:200-254): device state f32[n][obs_dim], ids
 * i32[n][K] (null: every action, K = n_actions) -> out_q f32[n][K], the advantage mean over the row's K ids; online
 * (target = 0) or target network.  1 <= K <= n_actions + 1. */
int prl_duel_q_values(prl_duel *duel, int n, const float *state, const int32_t *ids, int K, int target, float *out_q_dev,
                      void *stream);
int prl_duel_set_graph(prl_duel *duel, int enable);
int64_t prl_duel_last_launches(const prl_duel *duel);

/* ---- multi-head DQN / DoubleDQN (plain or conservative) ------------------------------------------
 * Replaces VanillaQValueMultiHeadNetwork.get_q_values (neural_networks/sequential_decision_making/q_value_networks.py:
 * 185-241), DeepTDLearning.forward / loss / learn_batch (policy_learners/sequential_decision_making/deep_td_learning.py:
 * 269-360), DeepQLearning / DoubleDQN.get_next_state_values (deep_q_learning.py:130-167, double_dqn.py:29-57) and, when
 * conservative, compute_cql_loss (utils/functional_utils/learning/loss_fn_utils.py:17-71), driven by PolicyLearner.learn
 * (prl_mhq_learn: sample -> round, `rounds` times) or called on a caller's batch (prl_mhq_learn_batch: one round,
 * PearlAgent.learn_batch / offline_learning).  The network maps a state to one Q value per action, Q(s) = W3 relu(W2
 * relu(W1 s + b1) + b2) + b3; a query slot holding id k reads Q(s)[k] exactly (the reference's bmm with a one-hot slot).
 * Per round:
 *   when (training_steps + 1) % target_update_freq == 0, FIRST target = tau * online + (1 - tau) * target;
 *   q_b = Q(s_b)[a_b]; y_b = V_b gamma (1 - terminated_b) + r_b with V_b = max over available next slots k of
 *   Q'(s'_b)[id_k] (DQN) or Q'(s'_b)[id_k*], k* = first argmax over available next slots of Q(s'_b)[id_k] (DoubleDQN);
 *   L = mean_b (q_b - y_b)^2, plus, when conservative, alpha cql with cql = mean_b logsumexp_k Q(s_b)[c_b[k]]
 *   - (1 / (B A)) sum_b [(A - 1) Q(s_b)[c_b[0]] + Q(s_b)[c_b[1]]] (the reference gathers the current-slot values with the
 *   ONE-HOT action, as prl_cql documents; c_b[k] are the current slots including padding, id 0, so padded slots add on
 *   one head column); one AdamW(amsgrad) step.  Reported loss: mean_b |q_b - y_b| (the Bellman error only).
 * 1 <= n_actions <= 255 (2 <= n_actions when conservative: A = 1 makes the reference's gather index out of range);
 * 2 max_batch max(obs_dim, hidden1, hidden2, n_actions) < 2^31 and param_count < 2^31 (32-bit element offsets);
 * param_count / workspace_bytes return -1 and create returns EINVAL beyond these.  Flat layout (fp32, row-major
 * [out][in], torch's parameter order): W1[h1][obs] b1 W2[h2][h1] b2 W3[A][h2] b3[A].  Sharded buffers, continuous-action
 * buffers, buffers of other obs_dim / n_actions, and batch / rounds above the configured maxima are rejected (EINVAL)
 * before any launch. */
typedef struct prl_mhq_cfg {
    int32_t obs_dim, n_actions, hidden1, hidden2;
    int32_t double_dqn;            /* 0: DeepQLearning, 1: DoubleDQN */
    int32_t conservative;          /* 1: is_conservative=True (CQL term with the per-call alpha) */
    int32_t target_update_freq, max_batch, max_rounds;
    double lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_mhq_cfg;
typedef struct prl_mhq prl_mhq;
int64_t prl_mhq_param_count(const prl_mhq_cfg *cfg);
int64_t prl_mhq_workspace_bytes(const prl_mhq_cfg *cfg);
/* w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq: device f32[param_count] owned by the caller (the argument order of
 * prl_dqn_create); adam_step: optimizer steps already taken (torch's `step`). */
int prl_mhq_create(prl_mhq **out, const prl_mhq_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                   float *max_exp_avg_sq, int64_t adam_step, void *workspace_dev);
int prl_mhq_destroy(prl_mhq *mhq);
int64_t prl_mhq_adam_step(const prl_mhq *mhq);
int prl_mhq_set_adam_step(prl_mhq *mhq, int64_t step);
/* New AdamW learning rate from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_mhq_set_lr(prl_mhq *mhq, double lr);
/* training_steps = the learner's count before the call (PolicyLearner.learn increments it before each round); alpha =
 * conservative_alpha (ignored unless conservative); out_loss_dev: device f32[rounds]; out_logical_dev (optional)
 * i32[rounds][batch] = sampled indices.  The ring stores no current action sets: every round uses the full set, as
 * B200ReplayBuffer.sample reports it. */
int prl_mhq_learn(prl_mhq *mhq, prl_buf *buf, int rounds, int batch, int64_t training_steps, double alpha,
                  float *out_loss_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action_id i32[batch], reward f32[batch],
 * terminated u8[batch]; curr_ids i32[batch][n_actions] (slot k of the current set, padding included; read only when
 * conservative), null = every action; next_ids i32[batch][n_actions] and next_count i32[batch] (slots at and beyond it
 * are unavailable), both null when every action is available next; training_steps = the count learn_batch sees
 * (agent.learn_batch does not advance it); out_loss_dev: device f32[1]. */
int prl_mhq_learn_batch(prl_mhq *mhq, int batch, const float *state, const int32_t *action_id, const float *reward,
                        const float *next_state, const uint8_t *terminated, const int32_t *curr_ids, const int32_t *next_ids,
                        const int32_t *next_count, int64_t training_steps, double alpha, float *out_loss_dev, void *stream);
/* Q(s)[a] for every action (DeepTDLearning.act, deep_td_learning.py:200-254): device state f32[n][obs_dim] ->
 * out_q f32[n][n_actions], online (target = 0) or target network. */
int prl_mhq_q_values(prl_mhq *mhq, int n, const float *state, int target, float *out_q_dev, void *stream);
int prl_mhq_set_graph(prl_mhq *mhq, int enable);
int64_t prl_mhq_last_launches(const prl_mhq *mhq);

/* ---- DeepSARSA ------------------------------------------------------------------------------------
 * Replaces DeepSARSA.get_next_state_values (policy_learners/sequential_decision_making/deep_sarsa.py:58-75) on
 * DeepTDLearning.forward / loss / learn_batch (deep_td_learning.py:269-360) with VanillaQValueNetwork.get_q_values
 * (neural_networks/sequential_decision_making/q_value_networks.py:152-174), driven by PolicyLearner.learn (prl_sarsa_learn:
 * sample -> round, `rounds` times, over a PRL_BUF_NEXT_ACTION buffer) or called on a caller's batch (prl_sarsa_learn_batch:
 * one round, PearlAgent.learn_batch).  Per round:
 *   when (training_steps + 1) % target_update_freq == 0, FIRST target = tau * online + (1 - tau) * target;
 *   q_b = Q(s_b, a_b); y_b = Q'(s'_b, a'_b) gamma (1 - terminated_b) + r_b with a'_b the committed next action (no max,
 *   the available sets take no part); L = mean_b (q_b - y_b)^2; one AdamW(amsgrad) step.  Reported loss: mean_b |q_b - y_b|.
 * 1 <= n_actions <= 255.  Flat layout as prl_dqn: W1[h1][obs + A] b1 W2[h2][h1] b2 W3[1][h2] b3.  Buffers without
 * PRL_BUF_NEXT_ACTION, sharded, continuous-action or mismatched buffers, and batch / rounds above the configured maxima
 * are rejected (EINVAL) before any launch.
 * The round is captured into a CUDA graph per (batch, buffer) and kept in a small cache (least recently used out), so an
 * on-policy loop whose batch follows the episode length replays the graph of a batch size it has seen. */
typedef struct prl_sarsa_cfg {
    int32_t obs_dim, n_actions, hidden1, hidden2;
    int32_t target_update_freq, max_batch, max_rounds;
    double lr, beta1, beta2, eps, weight_decay, gamma, tau;
} prl_sarsa_cfg;
typedef struct prl_sarsa prl_sarsa;
int64_t prl_sarsa_param_count(const prl_sarsa_cfg *cfg);
int64_t prl_sarsa_workspace_bytes(const prl_sarsa_cfg *cfg);
/* w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq: device f32[param_count] owned by the caller (the argument order of
 * prl_dqn_create); adam_step: optimizer steps already taken (torch's `step`). */
int prl_sarsa_create(prl_sarsa **out, const prl_sarsa_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                     float *max_exp_avg_sq, int64_t adam_step, void *workspace_dev);
int prl_sarsa_destroy(prl_sarsa *sarsa);
int64_t prl_sarsa_adam_step(const prl_sarsa *sarsa);
int prl_sarsa_set_adam_step(prl_sarsa *sarsa, int64_t step);
/* New AdamW learning rate from the next call on; every lr-dependent scalar travels in the per-call block: no re-capture. */
int prl_sarsa_set_lr(prl_sarsa *sarsa, double lr);
/* training_steps = the learner's count before the call (PolicyLearner.learn increments it before each round);
 * out_loss_dev: device f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices. */
int prl_sarsa_learn(prl_sarsa *sarsa, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss_dev,
                    int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state / next_state f32[batch][obs], action_id / next_action_id i32[batch] in
 * [0, n_actions), reward f32[batch], terminated u8[batch]; training_steps = the count learn_batch sees (agent.learn_batch
 * does not advance it); out_loss_dev: device f32[1]. */
int prl_sarsa_learn_batch(prl_sarsa *sarsa, int batch, const float *state, const int32_t *action_id, const float *reward,
                          const float *next_state, const int32_t *next_action_id, const uint8_t *terminated,
                          int64_t training_steps, float *out_loss_dev, void *stream);
/* Q(s, a) for every action: device state f32[n][obs_dim] -> out_q f32[n][n_actions], online (target = 0) or target. */
int prl_sarsa_q_values(prl_sarsa *sarsa, int n, const float *state, int target, float *out_q_dev, void *stream);
int prl_sarsa_set_graph(prl_sarsa *sarsa, int enable);
int64_t prl_sarsa_last_launches(const prl_sarsa *sarsa);
/* CUDA graphs captured by this handle so far (a batch size already in the graph cache adds none). */
int64_t prl_sarsa_graph_captures(const prl_sarsa *sarsa);

/* ---- PPO learner ------------------------------------------------------------------------------
 * Replaces ProximalPolicyOptimization.learn (policy_learners/sequential_decision_making/ppo.py:195-293):
 * prl_ppo_preprocess = preprocess_replay_buffer (state values, taken-action probabilities under the current
 * policy, GAE and truncated lambda returns over the whole rollout, time order), prl_ppo_learn =
 * PolicyLearner.learn (policy_learner.py:162-204) x ActorCriticBase.learn_batch (actor_critic_base.py:309-349):
 * clipped-surrogate actor step (ppo.py:152-184; VanillaActorNetwork softmax policy) then the state-value critic
 * step (critic_utils.py:139-167).  Flat parameter layouts (row-major [out][in]):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 W3[A][h2] b3      critic: W1[c1][obs] b1 W2[c2][c1] b2 W3[1][c2] b3 */
typedef struct prl_ppo_cfg {
    int32_t obs_dim, n_actions, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t max_batch, max_rounds;
    int64_t max_rollout;
    double actor_lr, critic_lr, beta1, beta2, eps, weight_decay, gamma, lam, epsilon, entropy_bonus;
} prl_ppo_cfg;
typedef struct prl_ppo prl_ppo;
int64_t prl_ppo_actor_param_count(const prl_ppo_cfg *cfg);
int64_t prl_ppo_critic_param_count(const prl_ppo_cfg *cfg);
int64_t prl_ppo_workspace_bytes(const prl_ppo_cfg *cfg);
int prl_ppo_create(prl_ppo **out, const prl_ppo_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                   float *critic_w, float *critic_m, float *critic_v, float *critic_vmax, int64_t adam_step,
                   void *workspace);
int prl_ppo_destroy(prl_ppo *ppo);
int64_t prl_ppo_adam_step(const prl_ppo *ppo);
int prl_ppo_set_graph(prl_ppo *ppo, int enable);
int64_t prl_ppo_last_launches(const prl_ppo *ppo);
/* outputs: device f32[len(buf)] each, index 0 = oldest stored transition; out_cut_dev (optional) u8[len]:
 * 1 where the transition is terminated or truncated (ends a GAE chain) */
int prl_ppo_preprocess(prl_ppo *ppo, prl_buf *buf, float *out_values_dev, float *out_action_probs_dev,
                       float *out_gae_dev, float *out_lam_return_dev, uint8_t *out_cut_dev, void *stream);
/* Rollout sharded over ranks by contiguous time chunks: re-run this chunk's GAE chains with V(next) of its newest
 * transition = `next_value` (first state value of the next, newer chunk) and the chain entering from there =
 * `incoming_gae` (that chunk's first gae).  Uses the rewards / flags staged by the last prl_ppo_preprocess.
 * Bit-identical to the unsharded computation. */
int prl_ppo_gae_redo(prl_ppo *ppo, const float *values_dev, float next_value, float incoming_gae,
                     float *out_gae_dev, float *out_lam_return_dev, void *stream);
/* gae / lam_return / action_probs: the arrays prl_ppo_preprocess produced; out_*_loss: device f32[rounds] */
int prl_ppo_learn(prl_ppo *ppo, prl_buf *buf, int rounds, int batch, const float *gae_dev,
                  const float *lam_return_dev, const float *action_probs_dev, float *out_actor_loss_dev,
                  float *out_critic_loss_dev, int32_t *out_logical_dev, void *stream);

/* ---- REINFORCE learner (state-value baseline) -------------------------------------------------------
 * Replaces REINFORCE.learn (policy_learners/sequential_decision_making/reinforce.py:179-208, losses :146-167) on top of
 * ActorCriticBase.learn_batch (actor_critic_base.py:309-366) and PolicyLearner.learn (policy_learner.py:162-204), with
 * use_critic=True, VanillaActorNetwork (softmax policy over every action, actor_networks.py:155-176) and
 * VanillaValueNetwork, two hidden layers each.  prl_reinforce_returns = the return pass: R = critic(next_state of the newest
 * transition) * (1 - terminated) + the rewards of every stored transition added newest -> oldest in fp32 (no discount, no
 * episode reset; every transition of the reference holds this one value).  prl_reinforce_learn = rounds x (sample -> actor
 * step on B * sum_j nlp_j (R - v_j), the reference's B x B broadcast -> critic step on mean((v - R)^2)), two AdamW(amsgrad)
 * states.  Flat parameter layouts (row-major [out][in]):
 *   actor : W1[h1][obs] b1 W2[h2][h1] b2 W3[A][h2] b3      critic: W1[c1][obs] b1 W2[c2][c1] b2 W3[1][c2] b3
 * 1 <= n_actions <= 255.  Continuous-action, mismatched and sharded buffers are rejected (EINVAL) before any launch. */
typedef struct prl_reinforce_cfg {
    int32_t obs_dim, n_actions, actor_h1, actor_h2, critic_h1, critic_h2;
    int32_t max_batch, max_rounds;
    double actor_lr, critic_lr, beta1, beta2, eps, weight_decay;
} prl_reinforce_cfg;
typedef struct prl_reinforce prl_reinforce;
int64_t prl_reinforce_actor_param_count(const prl_reinforce_cfg *cfg);
int64_t prl_reinforce_critic_param_count(const prl_reinforce_cfg *cfg);
int64_t prl_reinforce_workspace_bytes(const prl_reinforce_cfg *cfg);
int prl_reinforce_create(prl_reinforce **out, const prl_reinforce_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                         float *actor_vmax, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                         int64_t adam_step, void *workspace);
int prl_reinforce_destroy(prl_reinforce *rf);
int64_t prl_reinforce_adam_step(const prl_reinforce *rf);
/* New actor / critic AdamW learning rates from the next learn on.  Every lr-dependent scalar travels in the per-call
 * block: no re-capture, same handle. */
int prl_reinforce_set_lr(prl_reinforce *rf, double actor_lr, double critic_lr);
int prl_reinforce_set_graph(prl_reinforce *rf, int enable);
int64_t prl_reinforce_last_launches(const prl_reinforce *rf);
/* out_return_dev: device f32[2] = {R, the bootstrap term critic(s'_newest) * (1 - terminated)}.  Given the same
 * bootstrap term, R is bit-identical to the reference's fold. */
int prl_reinforce_returns(prl_reinforce *rf, prl_buf *buf, float *out_return_dev, void *stream);
/* return_dev: the array prl_reinforce_returns wrote (R = return_dev[0]); out_*_loss: device f32[rounds];
 * out_logical_dev (optional) i32[rounds][batch] = sampled indices */
int prl_reinforce_learn(prl_reinforce *rf, prl_buf *buf, int rounds, int batch, const float *return_dev,
                        float *out_actor_loss_dev, float *out_critic_loss_dev, int32_t *out_logical_dev, void *stream);

/* Device timing of the persistent learner kernel alone (CUDA events recorded on
 * the launch stream around the kernel); used by bench.py for the roofline line.
 * prl_dqn_last_kernel_ms synchronises on the end event. */
int prl_dqn_set_timing(prl_dqn *dqn, int enable);
/* Developer profiling: device int64[rounds][16] receiving SM-clock stamps of one CTA at
 * the phase boundaries of every round of the next prl_dqn_learn calls (NULL = off).  The
 * tensor-core group kernel stamps CTA $PRL_TC_PROF_CTA (default 0), the cooperative kernel CTA 0. */
int prl_dqn_set_profile(prl_dqn *dqn, long long *stamps_dev);
int prl_dqn_last_kernel_ms(prl_dqn *dqn, float *ms);

/* Self-test of the wgmma building block used by the learner kernels: one CTA computes
 * D[128][n] = A[128][k] * B[n][k]^T (device fp32 row-major arrays) with plain TF32 (passes = 1) or
 * the 3xTF32 split the learner uses for fp32 parity (passes = 3).  Test infrastructure hook. */
int prl_test_umma_gemm(const float *a_dev, const float *b_dev, float *d_dev, int n, int k, int passes,
                       void *stream);
/* Same product with the A operand in registers (RS form), B in shared memory;
 * k <= 64, n = 32 or a multiple of 64; `reps` is ignored. */
int prl_test_umma_gemm_ts(const float *a_dev, const float *b_dev, float *d_dev, int n, int k, int reps, void *stream);
/* General self-test: D[m][n] = A[m][k] * B[n][k]^T with m in {64,128} and a free operand chunk pitch
 * `lbo` (128 dense / 144 transposed-write friendly, see csrc/umma.cuh).  draw_dev receives the
 * product, row-major [m x n]. */
int prl_test_umma_gemm2(const float *a_dev, const float *b_dev, float *draw_dev, int m, int n, int k, int lbo,
                        void *stream);

/* ---- contraction engine of the actor-critic learners (SAC, PPO, TD3 / DDPG) --------------------------------
 * The dense layers of those learners (the torch matmuls of pearl/neural_networks/common/utils.py:mlp_block as used by
 * actor_networks.py / value_networks.py, forward and autograd backward) run as 3xTF32 wgmma tiles or as fp32 SIMT tiles:
 * engine 1 (default) uses the tensor-core tiles for products with at least 4096 output rows (a threshold not measured on H100), 0 = SIMT only,
 * 2 = tensor cores always.  Process-wide; read when a learner's round is launched or captured into its CUDA graph, so set it
 * before the first learn() of a learner. */
int prl_set_contraction_engine(int engine);
int prl_get_contraction_engine(void);
/* Test hook: one contraction of the three kinds the learners use, `nets` stacked problems contiguous in every operand.
 *   op 0  c[M x N]   = act(x W^T + bias)      a = x [M x K] (or [M x split] and a2 = [M x (K - split)]), b = W [N x K]
 *   op 1  c[M x K] (+)= dy W, masked          a = dy [M x N], b = W [N x K], mask [M x K] (keep where mask > 0)
 *   op 2  c[N x K]   = dy^T x, c_tail = dy^T 1  a = dy [M x N], b = x [M x K] (or split with a2)
 * engine: -1 library default, 0 SIMT, 1 automatic, 2 tensor cores always; 64 / 32: the shared-memory-operand form with that tile
 * width, 164 / 132: the register-operand form with tile width 64 / 32. */
int prl_test_contraction(int op, int engine, int M, int N, int K, const float *a, const float *b, const float *a2, int split,
                         const float *bias, const float *mask, int relu, int accumulate, float *c, float *c_tail, int nets,
                         void *stream);

/* ---- contextual bandit: LinearBandit (LinUCB) ------------------------------------------------------------------
 * Replaces LinearRegression.learn_batch / calculate_coefs / apply_discounting / forward / calculate_sigma
 * (neural_networks/contextual_bandit/linear_regression.py:192-270), LinearBandit.learn_batch / _maybe_apply_discounting
 * (policy_learners/contextual_bandits/linear_bandit.py:123-164), driven by PolicyLearner.learn (prl_cb_learn: sample ->
 * round, `rounds` times) or called on a caller's batch (prl_cb_learn_batch: one round, PearlAgent.learn_batch /
 * offline_learning), and the UCB scores of LinearBandit.act / get_scores (ucb_exploration.py:40-93, action_utils.py:150-158).
 * With x = state || action features (k = obs_dim + action_dim) and x1 = [1, x] (d = k + 1), per round:
 *   A += x1^T (x1 w), b += x1^T (y w), sum_weight += sum w   (fp32, the partial sums added in a fixed order);
 *   when discount_interval > 0 and (double)sum_weight - last_discount >= discount_interval: A, b *= gamma (when gamma < 1)
 *   and last_discount = sum_weight;  inv_A = inv(A + lambda I), coefs = inv_A b  (Gauss-Jordan with partial pivoting in
 *   fp64, rounded to fp32);  prediction = x1 . coefs with the new coefs.
 * d <= 128; l2_reg_lambda > 0 (the reference's pinv fallback is not implemented); workspace_bytes returns -1 and create
 * returns EINVAL beyond these.  Weights must be non-negative (not checked here): with a negative weight A + lambda I can
 * be singular, where the reference falls back to pinv and this solve returns non-finite values.  In learn, action_rep folds the stored id into the row: 1 = one-hot over action_dim =
 * n_actions columns, 2 = binary code, bit p of the id at column p (BinaryActionTensorRepresentationModule);
 * learn refuses action_rep 0.  Sharded buffers, continuous-action buffers, buffers of other obs_dim / n_actions, and
 * batch / rounds above the configured maxima are rejected (EINVAL) before any launch. */
typedef struct prl_cb_cfg {
    int32_t obs_dim, n_actions, action_dim;
    int32_t action_rep;            /* 0: none (learn_batch / scores only), 1: one-hot, 2: binary */
    int32_t max_batch, max_rounds;
    double l2_reg_lambda, gamma, discount_interval;
} prl_cb_cfg;
typedef struct prl_cb prl_cb;
int64_t prl_cb_workspace_bytes(const prl_cb_cfg *cfg);
/* A f32[d][d], b f32[d], sum_weight f32[1], inv_A f32[d][d], coefs f32[d], last_discount f64[1]: device memory owned by the
 * caller (the reference's buffers _A, _b, _sum_weight, _inv_A, _coefs and last_sum_weight_when_discounted). */
int prl_cb_create(prl_cb **out, const prl_cb_cfg *cfg, float *A, float *b, float *sum_weight, float *inv_A, float *coefs,
                  double *last_discount, void *workspace_dev);
int prl_cb_destroy(prl_cb *cb);
int prl_cb_set_graph(prl_cb *cb, int enable);
int64_t prl_cb_last_launches(const prl_cb *cb);
/* out_pred_dev / out_label_dev / out_weight_dev: device f32[rounds][batch] (label and weight may be null);
 * out_logical_dev (optional) i32[rounds][batch] = sampled indices.  Every stored transition has weight 1. */
int prl_cb_learn(prl_cb *cb, prl_buf *buf, int rounds, int batch, float *out_pred_dev, float *out_label_dev, float *out_weight_dev,
                 int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch: state f32[batch][obs_dim], action f32[batch][action_dim] (the represented action, used
 * as given), reward f32[batch], weight f32[batch] (null: every weight 1); out_pred_dev f32[batch]. */
int prl_cb_learn_batch(prl_cb *cb, int batch, const float *state, const float *action, const float *reward, const float *weight,
                       float *out_pred_dev, void *stream);
/* Scores of n states x n_space actions: state f32[n][obs_dim], act_feat f32[n_space][action_dim] (the represented actions of
 * the space); out_scores f32[n][n_space] = x1 . coefs (+ alpha sigma when with_sigma, sigma = sqrt(x1^T inv_A x1), NaN ->
 * 0); out_index (optional) i32[n] = first maximum over the positions where mask u8[n][n_space] is non-zero (mask null:
 * every position; 0 when none is). */
int prl_cb_scores(prl_cb *cb, int n, const float *state, int n_space, const float *act_feat, double alpha, int with_sigma,
                  const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream);
/* Thompson sampling, replacing ThompsonSamplingExplorationLinear.get_scores's default branch
 * (policy_learners/exploration_modules/contextual_bandits/thompson_sampling_exploration.py:63-72, MultivariateNormal(loc =
 * coefs, precision_matrix = A + lambda I).sample()) for both ridge learners (LinearBandit: d = feature_dim + 1;
 * NeuralLinearBandit: d = h2 + 1), on the device buffers A_dev f32[d][d] (symmetric) and coefs_dev f32[d]:
 * out_theta_dev f32[d] = coefs + U^-T eps with M = A + (float)lambda I formed in fp32 and factored M = U U^T (U upper
 * triangular) in fp64, for the caller's standard normal draws eps_dev f32[d].  1 <= d <= 128.  One CTA, no handle, no
 * host synchronisation.  out_status_dev i32[1] = 0, or 1 when M is not positive definite (theta is then unwritten; the
 * reference raises ValueError). */
int prl_cb_ts_sample(int d, double lambda, const float *A_dev, const float *coefs_dev, const float *eps_dev, float *out_theta_dev,
                     int32_t *out_status_dev, void *stream);
/* Thompson scores of n states x n_space actions (state, act_feat, mask and out_index as prl_cb_scores), exactly one of:
 *   theta_dev f32[d] (from prl_cb_ts_sample): out_scores = x1 . theta  (thompson_sampling_exploration.py:69-72);
 *   z_dev f32[n][n_space] (enable_efficient_sampling, lines 53-61): out_scores = mu + z sigma, rounded after the product
 *   and after the sum as torch.normal(mean = mu, std = sigma) computes it, mu = x1 . coefs, sigma = sqrt(x1^T inv_A x1);
 *   out_status_dev i32[1] = 1 when a sigma is NaN (torch.normal raises there), else 0.
 * out_status_dev may be null with theta. */
int prl_cb_ts_scores(prl_cb *cb, int n, const float *state, int n_space, const float *act_feat, const float *theta_dev,
                     const float *z_dev, const uint8_t *mask, float *out_scores, int32_t *out_index, int32_t *out_status_dev,
                     void *stream);

/* ---- contextual bandit: NeuralLinearBandit (neural LinUCB) -------------------------------------------------------
 * Replaces NeuralLinearBandit.learn_batch / act / get_scores (policy_learners/contextual_bandits/neural_linear_bandit.py)
 * over NeuralLinearRegression (neural_networks/contextual_bandit/neural_linear_regression.py) with two hidden layers.
 * Network input x = state (action_dim 0: state_features_only) or state || action features; nn_output = mlp_block(x,
 * [h1, h2], output_dim = h2) with ReLU, each layer of equal in / out width wrapped as x + layer(x) when skip.  Per round:
 *   forward with the current parameters; mu = nn_output . e2e weight (e2e) or [1, nn_output] . coefs (the coefs before
 *   this round's ridge update); p = sigmoid(mu) when sigmoid, else mu; loss = sum(w l(p, y)) / sum(w), l = mse (0),
 *   l1 (1) or binary cross-entropy (2, needs sigmoid); backward and one AdamW(amsgrad) step over the network (and the e2e
 *   weight when e2e); then the ridge of prl_cb (A, b, sum_weight, discounting, inv_A, coefs) on the pre-step nn_output.
 * Flat parameters w f32[param_count] in torch's parameters() order: W1[h1][f] b1 W2[h2][h1] b2 W3[h2][h2] b3, then the
 * e2e weight [h2]; m / v / vmax are the AdamW exp_avg / exp_avg_sq / max_exp_avg_sq of the same layout.  The ridge
 * buffers are as prl_cb_create's, with d = h2 + 1.  1 <= h2 <= 127; l2_reg_lambda > 0.  score_rows: rows the workspace
 * holds for prl_nlb_scores per chunk (0: max_batch). */
typedef struct prl_nlb_cfg {
    int32_t obs_dim, n_actions, action_dim;
    int32_t action_rep;            /* 0: none (state alone, or learn_batch / scores), 1: one-hot, 2: binary */
    int32_t h1, h2, skip, e2e;
    int32_t loss;                  /* 0: mse, 1: mae, 2: binary cross-entropy */
    int32_t sigmoid;               /* output activation: 0 linear, 1 sigmoid */
    int32_t max_batch, max_rounds, score_rows;
    double lr, beta1, beta2, eps, weight_decay;
    double l2_reg_lambda, gamma, discount_interval;
} prl_nlb_cfg;
typedef struct prl_nlb prl_nlb;
int64_t prl_nlb_param_count(const prl_nlb_cfg *cfg);
int64_t prl_nlb_workspace_bytes(const prl_nlb_cfg *cfg);
int prl_nlb_create(prl_nlb **out, const prl_nlb_cfg *cfg, float *w, float *m, float *v, float *vmax, int64_t adam_step, float *A,
                   float *b, float *sum_weight, float *inv_A, float *coefs, double *last_discount, void *workspace_dev);
int prl_nlb_destroy(prl_nlb *nlb);
int prl_nlb_set_graph(prl_nlb *nlb, int enable);
int prl_nlb_set_lr(prl_nlb *nlb, double lr);           /* from the next call on; no new capture */
int64_t prl_nlb_adam_step(const prl_nlb *nlb);
int prl_nlb_set_adam_step(prl_nlb *nlb, int64_t step);
int64_t prl_nlb_last_launches(const prl_nlb *nlb);
int64_t prl_nlb_graph_captures(const prl_nlb *nlb);   /* rounds captured into CUDA graphs so far */
/* out_pred_dev (the pre-step, post-activation predictions) / out_label_dev / out_weight_dev: device f32[rounds][batch]
 * (label and weight may be null); out_loss_dev / out_mu_dev f32[rounds]: the loss and the mean prediction of each round;
 * out_logical_dev (optional) i32[rounds][batch] = sampled indices.  Every stored transition has weight 1. */
int prl_nlb_learn(prl_nlb *nlb, prl_buf *buf, int rounds, int batch, float *out_pred_dev, float *out_label_dev,
                  float *out_weight_dev, float *out_loss_dev, float *out_mu_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch (as prl_cb_learn_batch; action null when action_dim is 0).  zero_weight != 0: the
 * weights sum to 0, so the round takes no optimizer step (the loss is 0 and the AdamW step count does not advance) and only
 * the ridge is updated, as the reference's short circuit; the caller decides it (the reference reads the sum on the host). */
int prl_nlb_learn_batch(prl_nlb *nlb, int batch, const float *state, const float *action, const float *reward, const float *weight,
                        int zero_weight, float *out_pred_dev, float *out_loss_dev, float *out_mu_dev, void *stream);
/* Scores of n states x n_space actions (state and act_feat as prl_cb_scores; act_feat may be null when action_dim is 0):
 * mu from the network's output as in a round, sigma = sqrt([1, nn_output]^T inv_A [1, nn_output]) (NaN -> 0);
 * mode 0 (act): mu + alpha sigma; 1: activation(mu + alpha sigma); 2: activation(mu) + alpha sigma (separate_uncertainty).
 * out_index as prl_cb_scores. */
int prl_nlb_scores(prl_nlb *nlb, int n, const float *state, int n_space, const float *act_feat, double alpha, int mode,
                   const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream);
/* Thompson scores of n states x n_space actions (arguments as prl_nlb_scores), replacing the default branch of
 * ThompsonSamplingExplorationLinear.get_scores (thompson_sampling_exploration.py:63-74) as NeuralLinearBandit.act /
 * get_scores call it (neural_linear_bandit.py:252-258, 292-313): [1, nn_output] . theta_dev (f32[h2 + 1], from
 * prl_cb_ts_sample on this handle's ridge buffers), through the output activation when activate (get_scores without
 * separate_uncertainty); act and separate_uncertainty's get_scores pass activate = 0. */
int prl_nlb_ts_scores(prl_nlb *nlb, int n, const float *state, int n_space, const float *act_feat, const float *theta_dev,
                      int activate, const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream);

/* ---- contextual bandit: NeuralBandit (SquareCB / FastCB / greedy) -------------------------------------------------
 * Replaces NeuralBandit.learn_batch / act / get_scores (policy_learners/contextual_bandits/neural_bandit.py) over
 * VanillaValueNetwork with two hidden layers and one output.  Network input x = state (action_dim 0: state_features_only)
 * or state || action features; p = mlp_block(x, [h1, h2], output_dim = 1) with ReLU.  Per round: forward with the current
 * parameters; loss = sum(w l(p, y)) / sum(w), l = mse (0) or l1 (1), with no short circuit (a zero sum gives inf / NaN);
 * backward and one AdamW(amsgrad) step over the network.  Flat parameters w f32[param_count] in torch's parameters()
 * order: W1[h1][f] b1 W2[h2][h1] b2 W3[1][h2] b3; m / v / vmax are the AdamW exp_avg / exp_avg_sq / max_exp_avg_sq of
 * the same layout.  score_rows: rows the workspace holds for scoring per chunk (0: max_batch). */
typedef struct prl_nb_cfg {
    int32_t obs_dim, n_actions, action_dim;
    int32_t action_rep;            /* 0: none (state alone, or learn_batch / scores), 1: one-hot, 2: binary */
    int32_t h1, h2;
    int32_t loss;                  /* 0: mse, 1: mae (l1) */
    int32_t max_batch, max_rounds, score_rows;
    double lr, beta1, beta2, eps, weight_decay;
} prl_nb_cfg;
typedef struct prl_nb prl_nb;
int64_t prl_nb_param_count(const prl_nb_cfg *cfg);
int64_t prl_nb_workspace_bytes(const prl_nb_cfg *cfg);
int prl_nb_create(prl_nb **out, const prl_nb_cfg *cfg, float *w, float *m, float *v, float *vmax, int64_t adam_step,
                  void *workspace_dev);
int prl_nb_destroy(prl_nb *nb);
int prl_nb_set_graph(prl_nb *nb, int enable);
int prl_nb_set_lr(prl_nb *nb, double lr);              /* from the next call on; no new capture */
int64_t prl_nb_adam_step(const prl_nb *nb);
int prl_nb_set_adam_step(prl_nb *nb, int64_t step);
int64_t prl_nb_last_launches(const prl_nb *nb);
int64_t prl_nb_graph_captures(const prl_nb *nb);     /* rounds captured into CUDA graphs so far */
/* out_pred_dev (the pre-step network output) / out_label_dev / out_weight_dev: device f32[rounds][batch] (label and weight
 * may be null); out_loss_dev f32[rounds]; out_logical_dev (optional) i32[rounds][batch] = sampled indices.  Every stored
 * transition has weight 1. */
int prl_nb_learn(prl_nb *nb, prl_buf *buf, int rounds, int batch, float *out_pred_dev, float *out_label_dev,
                 float *out_weight_dev, float *out_loss_dev, int32_t *out_logical_dev, void *stream);
/* One round on a dense device batch (as prl_nlb_learn_batch; action null when action_dim is 0, weight null: all 1;
 * weights of either sign). */
int prl_nb_learn_batch(prl_nb *nb, int batch, const float *state, const float *action, const float *reward, const float *weight,
                       float *out_pred_dev, float *out_loss_dev, void *stream);
/* The network's output over n states x n_space actions (state and act_feat as prl_nlb_scores) into out_scores_dev
 * f32[n][n_space]. */
int prl_nb_scores(prl_nb *nb, int n, const float *state, int n_space, const float *act_feat, float *out_scores_dev, void *stream);
/* act: the scores as prl_nb_scores into out_values_dev, then
 *   kind 0 (NoExploration): out_index_dev i32[n] = the first maximum of each state over the positions whose mask
 *          (u8[n][n_space], may be null) is non-zero, 0 when none is;
 *   kind 1 (SquareCB) / 2 (FastCB), n = 1: prl_nb_explore on the state's values; the mask is ignored, as the reference
 *          ignores it.
 * No host synchronisation. */
int prl_nb_act(prl_nb *nb, int n, const float *state, int n_space, const float *act_feat, int kind, double gamma, double lb,
               double ub, int clamp, const float *E_dev, const uint8_t *mask, float *out_values_dev, float *out_prob_dev,
               int32_t *out_index_dev, void *stream);
/* SquareCB / FastCB action choice of one state (squarecb_exploration.py act), in fp32 with gamma, lb and ub rounded to
 * fp32: values clamped to [lb, ub] when clamp (always for FastCB); the first maximum; p = 1 / (A + gamma gap) (SquareCB) or
 * (max - lb) / (A (max - lb) + gamma gap), 1 / A when max <= lb (FastCB); p[max] = 1 - the sum of the others; pn = p / sum p;
 * out_index_dev i32[1] = the first maximum of pn / E over E_dev f32[n_space], the exponential draws of torch's one-sample
 * multinomial.  out_prob_dev f32[n_space] (may be null) = pn.  Device pointers; no handle. */
int prl_nb_explore(int n_space, const float *values_dev, int kind, double gamma, double lb, double ub, int clamp, const float *E_dev,
                   float *out_prob_dev, int32_t *out_index_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PEARL_B200_H */
