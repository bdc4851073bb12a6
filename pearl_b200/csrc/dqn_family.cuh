// dqn_family.cuh — the host half shared by the single-network DQN-family learners (qrdqn.cu, cql.cu, dueling.cu): the
// per-call tail of the workspace and its staging, the graph cache, the launch bookkeeping and the learn / learn_batch
// entries.  No device code.
//
// A learner's handle derives from DqnRounds<Self, Call> and provides
//   cfg          its prl_*_cfg (obs_dim, n_actions, max_batch, max_rounds, target_update_freq, lr, beta1, beta2,
//                weight_decay)
//   round        static int round(Self *, prl_buf *buf, int B, cudaStream_t): one round launched (or captured) on the
//                stream, buf == null: the dense batch of the call block; it sets launches_per_round
//   kFn, kName   its C prefix ("prl_cql") and the name its buffer refusals use ("CQL")
// Call is the learner's per-call block; it holds `slots`, `out_loss` and `decay`.
#pragma once
#include "host_runtime.cuh"

namespace prl {

template <class Self, class Call>
struct DqnRounds {
    int32_t *slots, *logical;                 // [max_rounds][B] sampled ring slots, logical indices
    // per-call tail of the workspace: scal float2[MR] | target_on int32[MR] | call (8-byte aligned) | round_idx
    float2 *scal;
    int *target_on;
    Call *call;
    int *round_idx;
    size_t tail_bytes = 0;
    Stage stage;
    bool use_graph = true;
    cudaGraphExec_t graph_exec[2] = {nullptr, nullptr};   // [0] rounds from a replay buffer, [1] learn_batch on a dense batch
    int graph_batch[2] = {0, 0};
    const uint32_t *graph_buf = nullptr;
    int graph_dynamic = -1;
    int launches_per_round = 0;
    int64_t adam_step = 0, last_launches = 0;

    static size_t call_offset(int MR) { return ((size_t)MR * 12 + 7) / 8 * 8; }

    // slots | logical | tail: the end of the learner's carve list
    void carve_tail(Carve &w, int MR, int64_t B) {
        char *tail;
        w(slots, MR * B); w(logical, MR * B);
        tail_bytes = call_offset(MR) + sizeof(Call) + 4;
        w(tail, (int64_t)tail_bytes);
        if (!tail) return;
        scal = (float2 *)tail;
        target_on = (int *)(tail + (size_t)MR * 8);
        call = (Call *)(tail + call_offset(MR));
        round_idx = (int *)(call + 1);
    }

    // the end of *_create, once the workspace is carved: hands the handle out, or deletes it when the pinned buffers of
    // the staging cannot be made
    static int open(Self *s, Self **out) {
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
        for (cudaGraphExec_t g : s->graph_exec) if (g) cudaGraphExecDestroy(g);
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
    static int set_lr(Self *s, double lr) {
        PRL_REQUIRE(s, "null handle");
        PRL_REQUIRE(lr >= 0.0, "the learning rate must be non-negative");
        s->cfg.lr = lr;
        return PRL_OK;
    }
    static int set_graph(Self *s, int enable) {
        PRL_REQUIRE(s, "null handle");
        s->use_graph = enable != 0;
        return PRL_OK;
    }
    static int64_t last_launches_of(const Self *s) { return s ? s->last_launches : -1; }

    // PolicyLearner.learn: `rounds` rounds over `buf`, sampled here.  dense: the call block with the learner's own fields
    // filled in (its dense-batch pointers stay null).
    static int learn(Self *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss, int32_t *out_logical,
                     const Call &dense, void *stream_) {
        PRL_REQUIRE(s && buf && out_loss, "null argument");
        const auto &c = s->cfg;
        PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                    "%s needs a discrete-action buffer with obs_dim = %d and n_actions = %d", Self::kName, c.obs_dim, c.n_actions);
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: %s samples local buffers only", Self::kName);
        cudaStream_t st = (cudaStream_t)stream_;
        int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
        if (rc) return rc;
        rc = s->upload(rounds, training_steps + 1, out_loss, dense, st);   // PolicyLearner.learn counts the round first
        if (rc) return rc;
        return s->run(buf, rounds, batch, st);
    }

    // learn_batch: one round on the caller's dense batch, whose pointers `dense` holds
    static int learn_batch(Self *s, int batch, int64_t training_steps, float *out_loss, const Call &dense, void *stream_) {
        PRL_REQUIRE(batch > 0 && batch <= s->cfg.max_batch, "batch outside the configured maximum");
        cudaStream_t st = (cudaStream_t)stream_;
        int rc = s->upload(1, training_steps, out_loss, dense, st);
        if (rc) return rc;
        return s->run(nullptr, 1, batch, st);
    }

    // per-call tail (AdamW scalars of every round, target-update flags, decay, `dense`, pointers), uploaded on `st`.
    // steps0 = the training-step count the reference's learn_batch sees in round 0; round r updates the target when
    // (steps0 + r + 1) % target_update_freq == 0.
    int upload(int rounds, int64_t steps0, float *out_loss, const Call &dense, cudaStream_t st) {
        const auto &c = static_cast<Self *>(this)->cfg;
        char *h = nullptr;
        int rc = stage.wait(&h);
        if (rc) return rc;
        const int MR = c.max_rounds;
        float2 *hs = reinterpret_cast<float2 *>(h);
        int *on = reinterpret_cast<int *>(h + (size_t)MR * 8);
        for (int r = 0; r < rounds; r++) {
            hs[r] = adam_scal(c.lr, c.beta1, c.beta2, adam_step + r + 1);
            on[r] = (steps0 + r + 1) % c.target_update_freq == 0 ? 1 : 0;
        }
        Call *hc = reinterpret_cast<Call *>(h + call_offset(MR));
        *hc = dense;
        hc->slots = slots; hc->out_loss = out_loss;
        hc->decay = (float)(1.0 - c.lr * c.weight_decay);
        *reinterpret_cast<int *>(hc + 1) = 0;
        return stage.send(scal, tail_bytes, st);
    }

    // `rounds` rounds: replays of the graph captured for this (batch, buffer, dynamic-action flag), or eager launches
    int run(prl_buf *buf, int rounds, int batch, cudaStream_t st) {
        Self *s = static_cast<Self *>(this);
        const int g = buf ? 0 : 1;
        const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
        if (use_graph) {
            if (!graph_exec[g] || graph_batch[g] != batch || (buf && (graph_buf != buf->records || graph_dynamic != dynamic))) {
                int rc = capture_graph(&graph_exec[g], Self::kFn, [&](cudaStream_t cs) { return Self::round(s, buf, batch, cs); });
                if (rc) return rc;
                graph_batch[g] = batch;
                if (buf) { graph_buf = buf->records; graph_dynamic = dynamic; }
            }
            for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(graph_exec[g], st));
        } else {
            for (int r = 0; r < rounds; r++) {
                int rc = Self::round(s, buf, batch, st);
                if (rc) return rc;
            }
        }
        PRL_CUDA(cudaGetLastError());
        adam_step += rounds;
        last_launches = (int64_t)launches_per_round * rounds;
        return PRL_OK;
    }
};

}  // namespace prl
