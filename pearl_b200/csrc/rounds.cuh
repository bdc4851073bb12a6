// rounds.cuh — the host half shared by every learner whose step is one fixed launch sequence per round (qrdqn.cu,
// cql.cu, dueling.cu, multihead.cu, sarsa.cu, sac.cu, sac_discrete.cu, td3.cu, iql.cu, ppo.cu, reinforce.cu, rc_safety.cu
// and the bandits): the per-call tail of the workspace and its staging, the cache of captured rounds, the launch
// bookkeeping and the learn / learn_batch entries; and, in FlatQ, the setup of the Q learners' handles over flat
// parameter and AdamW vectors.  No device code.
//
// A learner's handle derives from Rounds<Self, Call> and provides
//   cfg          its prl_*_cfg (max_batch, max_rounds, beta1, beta2, and the learning rates)
//   round        static int round(Self *, prl_buf *buf, int B, cudaStream_t): one round launched (or captured) on the
//                stream, buf == null: the dense batch of the call block; it sets launches_per_round
//   kFn          its C prefix ("prl_cql"), which error messages name
// and, where the defaults below do not fit,
//   kScal        K, the AdamW step scalars per round, one per optimizer (default 1)
//   kCounters    device round counters after the call block, zeroed every call (default 1: round_idx)
//   kTargetOn    a per-round target-update flag after the scalars (the DQN family; needs cfg.target_update_freq)
//   kGraphs      captured rounds kept (default 1)
//   kName        the name the default buffer_ok refusals use
//   lr(k)        the k-th learning rate, which the default scalars and set_lr use
//   fill_call    the learner's own fields of the call block (decay factors)
//   buffer_ok    the buffer refusals of learn (default: a local discrete-action buffer of matching dimensions)
//   variant(r)   which launch sequence round r runs (default 0), round_variant to launch it, fill_scal for the scalars
// Call is the learner's per-call block; it holds `slots`.
#pragma once
#include <new>

#include "host_runtime.cuh"

namespace prl {

// What a captured round bakes in: the buffer's storage and record layout (passed by value to the load kernels) and its
// flags (some loads take the dynamic-action flag as an argument), the batch and the launch sequence.  These are all the
// buffer fields a round reads; occupancy is read only by the sampling before it.  A buffer's storage is a caller-owned
// tensor whose address a new buffer may reuse, so the address alone does not identify what was captured.
// records == null: the dense batch of the call block.
struct GraphKey {
    const uint32_t *records;
    prl_buf_layout lay;
    uint32_t flags;
    int batch, variant;

    static GraphKey of(const prl_buf *buf, int batch, int variant) {
        GraphKey k;
        memset(&k, 0, sizeof(k));
        if (buf) { k.records = buf->records; k.lay = buf->lay; k.flags = buf->desc.flags; }
        k.batch = batch; k.variant = variant;
        return k;
    }
    bool operator==(const GraphKey &o) const {
        return records == o.records && flags == o.flags && batch == o.batch && variant == o.variant && memcmp(&lay, &o.lay, sizeof(lay)) == 0;
    }
};

// Captured rounds by key; a miss takes a free entry or evicts the least recently used one.  Each entry keeps the launch
// count of the round it holds.
struct GraphCache {
    struct Entry {
        GraphKey key;
        cudaGraphExec_t exec;
        int launches;
        int64_t used;
    };
    Entry *e = nullptr;
    int n = 0;
    int64_t uses = 0, captures = 0;

    GraphCache() = default;
    GraphCache(const GraphCache &) = delete;
    GraphCache &operator=(const GraphCache &) = delete;
    ~GraphCache() {
        for (int i = 0; i < n; i++) if (e[i].exec) cudaGraphExecDestroy(e[i].exec);
        delete[] e;
    }
    bool open(int entries) {
        e = new (std::nothrow) Entry[entries]();
        n = e ? entries : 0;
        return e != nullptr;
    }
    // the entry of `key`, captured by capture(&exec) (which returns the round's launch count in *launches) on a miss
    template <class Capture>
    int get(const GraphKey &key, Entry **out, Capture &&capture) {
        Entry *hit = nullptr;
        for (int i = 0; i < n && !hit; i++) if (e[i].exec && e[i].key == key) hit = &e[i];
        if (!hit) {
            hit = &e[0];
            for (int i = 0; i < n; i++) {
                if (!e[i].exec) { hit = &e[i]; break; }
                if (e[i].used < hit->used) hit = &e[i];
            }
            // capture_graph releases the evicted graph (freed once its launches in flight complete)
            int rc = capture(&hit->exec, &hit->launches);
            if (rc) return rc;
            hit->key = key;
            captures++;
        }
        hit->used = ++uses;
        *out = hit;
        return PRL_OK;
    }
};

template <class Self, class Call>
struct Rounds {
    static constexpr int kScal = 1, kCounters = 1, kGraphs = 1;
    static constexpr bool kTargetOn = false;

    int32_t *slots, *logical;                 // [max_rounds][B] sampled ring slots, logical indices
    // per-call tail of the workspace: scal float2[K][MR] | target_on int32[MR] (kTargetOn) | call (8-byte aligned) |
    // round counters int32[kCounters]
    float2 *scal;
    int *target_on;
    Call *call;
    int *round_idx;
    size_t tail_bytes = 0;
    Stage stage;
    GraphCache graphs;
    bool use_graph = true;
    int launches_per_round = 0;
    int64_t adam_step = 0, last_launches = 0;
    int64_t steps0 = 0;                       // the training-step count round 0 of the current call sees

    static size_t call_offset(int MR) { return ((size_t)MR * (8 * Self::kScal + (Self::kTargetOn ? 4 : 0)) + 7) / 8 * 8; }

    // slots | logical | tail: the end of the learner's carve list
    void carve_tail(Carve &w, int MR, int64_t B) {
        char *tail;
        w(slots, MR * B); w(logical, MR * B);
        tail_bytes = call_offset(MR) + sizeof(Call) + 4 * Self::kCounters;
        w(tail, (int64_t)tail_bytes);
        if (!tail) return;
        scal = (float2 *)tail;
        target_on = (int *)(tail + (size_t)MR * 8 * Self::kScal);
        call = (Call *)(tail + call_offset(MR));
        round_idx = (int *)(call + 1);
    }

    // the end of *_create, once the workspace is carved: hands the handle out, or deletes it when the pinned buffers of
    // the staging or the graph cache cannot be made
    static int open(Self *s, Self **out) {
        if (!s->graphs.open(Self::kGraphs)) {
            delete s;
            return fail(PRL_ENOMEM, "out of host memory");
        }
        const cudaError_t e = s->stage.open(s->tail_bytes);
        if (e != cudaSuccess) {
            delete s;
            return fail(PRL_ECUDA, "%s_create: %s", Self::kFn, cudaGetErrorString(e));
        }
        *out = s;
        return PRL_OK;
    }
    static int destroy(Self *s) {
        if (!s) return PRL_OK;
        s->stage.close();
        delete s;
        return PRL_OK;
    }

    static int64_t adam_step_of(const Self *s) { return s ? s->adam_step : -1; }
    static int set_adam_step(Self *s, int64_t step) {
        PRL_REQUIRE(s, "null handle");
        PRL_REQUIRE(step >= 0, "the AdamW step count must be non-negative");
        s->adam_step = step;
        return PRL_OK;
    }
    // the first sizeof...(lr) learning rates, in lr(k) order
    template <class... Lr>
    static int set_lr(Self *s, Lr... lr) {
        PRL_REQUIRE(s, "null handle");
        const double v[] = {lr...};
        for (double x : v)
            PRL_REQUIRE(x >= 0.0, sizeof...(Lr) == 1 ? "the learning rate must be non-negative" : "learning rates must be non-negative");
        for (int k = 0; k < (int)sizeof...(Lr); k++) s->lr(k) = v[k];
        return PRL_OK;
    }
    static int set_graph(Self *s, int enable) {
        PRL_REQUIRE(s, "null handle");
        s->use_graph = enable != 0;
        return PRL_OK;
    }
    static int64_t last_launches_of(const Self *s) { return s ? s->last_launches : -1; }

    int buffer_ok(const prl_buf *buf) const {
        const auto &c = static_cast<const Self *>(this)->cfg;
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                    "%s needs a discrete-action buffer with obs_dim = %d and n_actions = %d", Self::kName, c.obs_dim, c.n_actions);
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: %s samples local buffers only", Self::kName);
        return PRL_OK;
    }

    // PolicyLearner.learn: `rounds` rounds over `buf`, sampled here.  call: the learner's fields of the call block (its
    // dense-batch pointers stay null).
    static int learn(Self *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, int32_t *out_logical, const Call &call,
                     void *stream_) {
        const auto &c = s->cfg;
        PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
        int rc = s->buffer_ok(buf);
        if (rc) return rc;
        cudaStream_t st = (cudaStream_t)stream_;
        rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
        if (rc) return rc;
        rc = s->upload(rounds, training_steps + 1, call, st);   // PolicyLearner.learn counts the round first
        if (rc) return rc;
        return s->run(buf, rounds, batch, st);
    }

    // learn_batch: one round on the caller's dense batch, whose pointers `call` holds
    static int learn_batch(Self *s, int batch, int64_t training_steps, const Call &call, void *stream_) {
        PRL_REQUIRE(batch > 0 && batch <= s->cfg.max_batch, "batch outside the configured maximum");
        cudaStream_t st = (cudaStream_t)stream_;
        int rc = s->upload(1, training_steps, call, st);
        if (rc) return rc;
        return s->run(nullptr, 1, batch, st);
    }

    double &lr(int) { return static_cast<Self *>(this)->cfg.lr; }
    void fill_call(Call &) const {}
    int variant(int) const { return 0; }
    int round_variant(prl_buf *buf, int B, int, cudaStream_t st) { return Self::round(static_cast<Self *>(this), buf, B, st); }
    // default scalars: the K learning rates at AdamW step adam_step + r + 1
    void fill_scal(float2 *hs, int rounds) {
        Self *s = static_cast<Self *>(this);
        const int MR = s->cfg.max_rounds;
        for (int k = 0; k < Self::kScal; k++)
            for (int r = 0; r < rounds; r++) hs[(size_t)k * MR + r] = adam_scal(s->lr(k), s->cfg.beta1, s->cfg.beta2, adam_step + r + 1);
    }

    // per-call tail (AdamW scalars of every round, target-update flags, `call`, counters), uploaded on `st`.
    // first = the training-step count the reference's learn_batch sees in round 0; round r updates the target when
    // (first + r + 1) % target_update_freq == 0.
    int upload(int rounds, int64_t first, const Call &callv, cudaStream_t st) {
        Self *s = static_cast<Self *>(this);
        const int MR = s->cfg.max_rounds;
        char *h = nullptr;
        int rc = stage.wait(&h);
        if (rc) return rc;
        steps0 = first;
        s->fill_scal(reinterpret_cast<float2 *>(h), rounds);
        if constexpr (Self::kTargetOn) {
            int *on = reinterpret_cast<int *>(h + (size_t)MR * 8 * Self::kScal);
            for (int r = 0; r < rounds; r++) on[r] = (first + r + 1) % s->cfg.target_update_freq == 0 ? 1 : 0;
        }
        Call *hc = reinterpret_cast<Call *>(h + call_offset(MR));
        *hc = callv;
        hc->slots = slots;
        s->fill_call(*hc);
        memset(hc + 1, 0, 4 * Self::kCounters);
        return stage.send(scal, tail_bytes, st);
    }

    // `rounds` rounds: replays of the graph cached for each round's key, captured on a miss, or eager launches
    int run(prl_buf *buf, int rounds, int batch, cudaStream_t st) {
        Self *s = static_cast<Self *>(this);
        int64_t launches = 0;
        GraphCache::Entry *g = nullptr;
        for (int r = 0; r < rounds; r++) {
            const int v = s->variant(r);
            if (!use_graph) {
                int rc = s->round_variant(buf, batch, v, st);
                if (rc) return rc;
                launches += launches_per_round;
                continue;
            }
            if (!g || g->key.variant != v) {
                int rc = graphs.get(GraphKey::of(buf, batch, v), &g, [&](cudaGraphExec_t *exec, int *n) {
                    int rc2 = capture_graph(exec, Self::kFn, [&](cudaStream_t cs) { return s->round_variant(buf, batch, v, cs); });
                    *n = launches_per_round;
                    return rc2;
                });
                if (rc) return rc;
            }
            PRL_CUDA(cudaGraphLaunch(g->exec, st));
            launches += g->launches;
        }
        PRL_CUDA(cudaGetLastError());
        adam_step += rounds;
        last_launches = launches;
        return PRL_OK;
    }
};

// The handle of a Q learner bound to caller-owned flat vectors: its parameters, the target's and the three AdamW states
// (cql.cu, dueling.cu, multihead.cu, sarsa.cu).  Self provides, besides what Rounds asks for,
//   check        static int check(const Cfg *): the configuration refusals
//   layout       static void layout(Self *): the parameter offsets and P from cfg
//   carve        static int64_t carve(Self *, void *base): the workspace in order; base == null: only its size
// Call holds `decay`, which fill_call sets.
template <class Self, class Call, class Cfg>
struct FlatQ : Rounds<Self, Call> {
    static constexpr bool kTargetOn = true;
    Cfg cfg;
    int P;
    float *q, *q_t, *q_m, *q_v, *q_x;         // online, target, exp_avg, exp_avg_sq, max_exp_avg_sq

    void fill_call(Call &k) const { k.decay = (float)(1.0 - cfg.lr * cfg.weight_decay); }

    static int64_t param_count(const Cfg *c) {
        if (Self::check(c)) return -1;
        Self t; t.cfg = *c; Self::layout(&t);
        return t.P;
    }
    static int64_t workspace_bytes(const Cfg *c) {
        if (Self::check(c)) return -1;
        Self t; t.cfg = *c; Self::layout(&t);
        return Self::carve(&t, nullptr);
    }
    static int create(Self **out, const Cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq,
                      int64_t adam_step, void *workspace) {
        PRL_REQUIRE(out && w && w_target && exp_avg && exp_avg_sq && max_exp_avg_sq && workspace, "null argument");
        int rc = Self::check(cfg);
        if (rc) return rc;
        Self *s = new (std::nothrow) Self();
        if (!s) return fail(PRL_ENOMEM, "out of host memory");
        s->cfg = *cfg;
        Self::layout(s);
        s->q = w; s->q_t = w_target; s->q_m = exp_avg; s->q_v = exp_avg_sq; s->q_x = max_exp_avg_sq;
        s->adam_step = adam_step;
        Self::carve(s, workspace);
        return Self::open(s, out);
    }
};

}  // namespace prl
