// replay_buffer.cu — GPU-resident ring replay buffer, MT19937-exact sampler,
// gather.  Replaces pearl/replay_buffers/{tensor_based,basic}_replay_buffer.py
// (see include/pearl_b200.h for the per-function reference citations).
#include <stdarg.h>

#include <new>

#include <algorithm>
#include <thread>
#include <vector>

#include "common.cuh"
#include "sampler.cuh"

namespace prl {
thread_local char g_err[512] = "";
}
using namespace prl;

// --------------------------------------------------------------------------
// library
// --------------------------------------------------------------------------
extern "C" int prl_abi_version(void) { return PRL_ABI_VERSION; }
extern "C" const char *prl_last_error(void) { return g_err; }

namespace prl { cudaError_t gemm_tc_prepare(); }   // gemm_tc.cu: opt the tensor-core contraction kernels into > 48 KB of shared memory

extern "C" int prl_init(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(PRL_EUNSUPPORTED, "no CUDA device (%s); libpearlb200 has no CPU path",
                    e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
    PRL_REQUIRE(device >= 0 && device < n, "device %d out of range (0..%d)", device, n - 1);
    PRL_CUDA(cudaSetDevice(device));
    cudaDeviceProp p;
    PRL_CUDA(cudaGetDeviceProperties(&p, device));
    if (p.major != 9)
        return fail(PRL_EUNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only",
                    device, p.major, p.minor);
    PRL_CUDA(prl::gemm_tc_prepare());
    return PRL_OK;
}

extern "C" int prl_sm_count(void) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return n;
}

// --------------------------------------------------------------------------
// layout
// --------------------------------------------------------------------------
extern "C" int prl_buf_layout_of(const prl_buf_desc *d, prl_buf_layout *out) {
    PRL_REQUIRE(d && out, "null argument");
    PRL_REQUIRE(d->capacity > 0 && d->capacity < (1ll << 31), "capacity must be in [1, 2^31)");
    PRL_REQUIRE(d->obs_dim > 0, "obs_dim must be positive");
    const bool disc = d->flags & PRL_BUF_DISCRETE, cont = d->flags & PRL_BUF_CONTINUOUS;
    PRL_REQUIRE(disc != cont, "exactly one of PRL_BUF_DISCRETE / PRL_BUF_CONTINUOUS");
    if (disc) PRL_REQUIRE(d->n_actions > 0 && d->n_actions <= 255, "n_actions must be in [1,255]");
    if (cont) PRL_REQUIRE(d->act_dim > 0, "act_dim must be positive");
    if (d->flags & PRL_BUF_DYNAMIC_ACTIONS) PRL_REQUIRE(disc, "dynamic action sets need a discrete space");
    if (d->flags & PRL_BUF_NEXT_ACTION) PRL_REQUIRE(disc, "a committed next action needs a discrete space");
    const int obs_p = round_up(d->obs_dim, 4);
    prl_buf_layout l;
    l.off_state = 0;
    l.off_next_state = obs_p;
    l.off_action = 2 * obs_p;
    l.act_words = disc ? 1 : d->act_dim;
    l.off_reward = l.off_action + l.act_words;
    l.off_flags = l.off_reward + 1;
    l.off_avail = l.off_flags + 1;
    int words = l.off_avail;
    if (d->flags & PRL_BUF_DYNAMIC_ACTIONS) words += (d->n_actions + 3) / 4;
    if (d->flags & PRL_BUF_COST) words += 1;      // the cost word goes last: no offset above moves
    l.record_words = round_up(words, 4);
    l.storage_bytes = d->capacity * (int64_t)l.record_words * 4;
    *out = l;
    return PRL_OK;
}

// the cost word of a PRL_BUF_COST record: right after the dynamic action ids (or after the flags word); -1 without costs
static int cost_word(const prl_buf_desc *d) {
    if (!(d->flags & PRL_BUF_COST)) return -1;
    prl_buf_layout l;
    prl_buf_layout_of(d, &l);
    return l.off_avail + ((d->flags & PRL_BUF_DYNAMIC_ACTIONS) ? (d->n_actions + 3) / 4 : 0);
}

extern "C" int prl_buf_cost_offset(const prl_buf_desc *d, int32_t *out) {
    PRL_REQUIRE(d && out, "null argument");
    prl_buf_layout l;
    const int rc = prl_buf_layout_of(d, &l);
    if (rc) return rc;
    PRL_REQUIRE(d->flags & PRL_BUF_COST, "the descriptor has no PRL_BUF_COST: its records store no cost");
    *out = cost_word(d);
    return PRL_OK;
}

// --------------------------------------------------------------------------
// create / destroy / occupancy
// --------------------------------------------------------------------------
static const int64_t kStageBytes = 8ll << 20;  // per pinned staging buffer

extern "C" int prl_buf_create(prl_buf **out, const prl_buf_desc *desc, void *storage_dev,
                              uint32_t *mt_state_dev) {
    PRL_REQUIRE(out && desc && storage_dev && mt_state_dev, "null argument");
    PRL_REQUIRE(((uintptr_t)storage_dev & 15) == 0, "storage must be 16-byte aligned");
    prl_buf_layout lay;
    int rc = prl_buf_layout_of(desc, &lay);
    if (rc) return rc;
    prl_buf *b = new (std::nothrow) prl_buf();
    if (!b) return fail(PRL_ENOMEM, "out of host memory");
    b->desc = *desc;
    b->lay = lay;
    b->records = (uint32_t *)storage_dev;
    b->mt_state = mt_state_dev;
    b->len = 0;
    b->write_pos = 0;
    b->stage[0] = b->stage[1] = nullptr;
    b->stage_records = 0;
    b->stage_next = 0;
    b->shard_rank = 0; b->shard_world = 1; b->g_pushed = 0;
    cudaGetDevice(&b->device);
    // never leave the MT19937 stream all-zero (it twists to zeros for ever: the set-branch sampler would then
    // spin on duplicates): a distinct default stream per buffer until the caller seeds / hands over a state
    static uint32_t created = 0;
    const uint32_t key[2] = {0x9e3779b9u, ++created};
    rc = prl_rng_seed(b, key, 2, nullptr);
    if (rc) { delete b; return rc; }
    *out = b;
    return PRL_OK;
}

extern "C" int prl_buf_destroy(prl_buf *b) {
    if (!b) return PRL_OK;
    for (int i = 0; i < 2; i++)
        if (b->stage[i]) {
            cudaEventSynchronize(b->stage_done[i]);
            cudaEventDestroy(b->stage_done[i]);
            cudaFreeHost(b->stage[i]);
        }
    delete b;
    return PRL_OK;
}

extern "C" int64_t prl_buf_len(const prl_buf *b) { return b ? b->len : 0; }
extern "C" int64_t prl_buf_capacity(const prl_buf *b) { return b ? b->desc.capacity : 0; }
extern "C" int64_t prl_buf_head(const prl_buf *b) {
    if (!b) return 0;
    int64_t h = b->write_pos - b->len;
    return h < 0 ? h + b->desc.capacity : h;
}
extern "C" int prl_buf_clear(prl_buf *b) {
    PRL_REQUIRE(b, "null buffer");
    b->len = 0;
    b->write_pos = 0;
    return PRL_OK;
}
extern "C" int prl_buf_set_occupancy(prl_buf *b, int64_t len, int64_t head) {
    PRL_REQUIRE(b, "null buffer");
    PRL_REQUIRE(len >= 0 && len <= b->desc.capacity, "len out of range");
    PRL_REQUIRE(head >= 0 && head < b->desc.capacity, "head out of range");
    b->len = len;
    b->write_pos = (head + len) % b->desc.capacity;
    return PRL_OK;
}

// --------------------------------------------------------------------------
// push
// --------------------------------------------------------------------------
static inline uint32_t f2u(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}

static int ensure_staging(prl_buf *b) {
    if (b->stage[0]) return PRL_OK;
    int64_t rec_bytes = (int64_t)b->lay.record_words * 4;
    int64_t n = kStageBytes / rec_bytes;
    if (n < 1) n = 1;
    for (int i = 0; i < 2; i++) {
        PRL_CUDA(cudaHostAlloc((void **)&b->stage[i], n * rec_bytes, cudaHostAllocDefault));
        PRL_CUDA(cudaEventCreateWithFlags(&b->stage_done[i], cudaEventDisableTiming));
    }
    b->stage_records = n;
    return PRL_OK;
}

// next_action: the committed next action ids of a PRL_BUF_NEXT_ACTION buffer (the *_sarsa entries), null for every other
// buffer; a push that would store id 0 for it, or drop it, is refused
static int check_next_action(const prl_buf *b, const void *next_action) {
    PRL_REQUIRE(b, "null buffer");
    if (b->desc.flags & PRL_BUF_NEXT_ACTION)
        PRL_REQUIRE(next_action, "the buffer stores a committed next action (PRL_BUF_NEXT_ACTION): push with the *_sarsa entries");
    else
        PRL_REQUIRE(!next_action, "next actions given for a buffer created without PRL_BUF_NEXT_ACTION");
    return PRL_OK;
}

// cost: the costs of a PRL_BUF_COST buffer (the *_cost entries), null for every other buffer
static int check_cost(const prl_buf *b, const void *cost) {
    PRL_REQUIRE(b, "null buffer");
    if (b->desc.flags & PRL_BUF_COST)
        PRL_REQUIRE(cost, "the buffer stores costs (PRL_BUF_COST): push with the *_cost entries");
    else
        PRL_REQUIRE(!cost, "costs given for a buffer created without PRL_BUF_COST");
    return PRL_OK;
}

static int check_push_args(const prl_buf *b, int64_t n, const void *state, const void *action,
                           const void *reward, const void *terminated, const void *truncated,
                           const void *ids, const void *cnt, const void *next_action, const void *cost) {
    PRL_REQUIRE(b, "null buffer");
    PRL_REQUIRE(n >= 0, "negative count");
    int rc = check_next_action(b, next_action);
    if (rc) return rc;
    rc = check_cost(b, cost);
    if (rc) return rc;
    if (n == 0) return PRL_OK;
    PRL_REQUIRE(state && action && reward && terminated && truncated, "null field array");
    PRL_REQUIRE((ids == nullptr) == (cnt == nullptr), "next_avail_ids and next_avail_cnt go together");
    if (ids)
        PRL_REQUIRE(b->desc.flags & PRL_BUF_DYNAMIC_ACTIONS,
                    "buffer was created without PRL_BUF_DYNAMIC_ACTIONS");
    return PRL_OK;
}

// pack transitions [i0, i0 + m) of struct-of-arrays host sources into m consecutive records at `st` (pure CPU)
static void pack_records_host(const prl_buf *b, uint32_t *st, int64_t i0, int64_t m, const float *state, const void *action,
                              const float *reward, const float *next_state, const uint8_t *terminated, const uint8_t *truncated,
                              const uint8_t *next_avail_ids, const int32_t *next_avail_cnt, const int32_t *next_action,
                              const float *cost) {
    const prl_buf_layout &L = b->lay;
    const int obs = b->desc.obs_dim, A = b->desc.n_actions, W = L.record_words, off_cost = cost_word(&b->desc);
    for (int64_t i = 0; i < m; i++) {
        const int64_t s = i0 + i;
        uint32_t *r = st + i * W;
        memcpy(r + L.off_state, state + s * obs, 4 * obs);
        for (int p = obs; p < L.off_next_state; p++) r[p] = 0;
        if (next_state)
            memcpy(r + L.off_next_state, next_state + s * obs, 4 * obs);
        else
            memset(r + L.off_next_state, 0, 4 * obs);
        for (int p = L.off_next_state + obs; p < L.off_action; p++) r[p] = 0;
        if (b->desc.flags & PRL_BUF_DISCRETE)
            r[L.off_action] = (uint32_t)((const int32_t *)action)[s];
        else
            memcpy(r + L.off_action, (const float *)action + s * L.act_words, 4 * L.act_words);
        r[L.off_reward] = f2u(reward[s]);
        uint32_t cnt = (b->desc.flags & PRL_BUF_DISCRETE) ? (uint32_t)A : 0u;
        if (next_avail_cnt) cnt = (uint32_t)next_avail_cnt[s];
        r[L.off_flags] = (terminated[s] ? 1u : 0u) | (truncated[s] ? 2u : 0u) | (cnt << 8) |
                         (next_action ? (uint32_t)next_action[s] << 24 : 0u);
        for (int p = L.off_avail; p < W; p++) r[p] = 0;
        if (b->desc.flags & PRL_BUF_DYNAMIC_ACTIONS) {
            uint8_t *ids = (uint8_t *)(r + L.off_avail);
            if (next_avail_ids)
                for (uint32_t a = 0; a < cnt && a < (uint32_t)A; a++) ids[a] = next_avail_ids[s * A + a];
            else
                for (int a = 0; a < A; a++) ids[a] = (uint8_t)a;
        }
        if (cost) r[off_cost] = f2u(cost[s]);
    }
}

// ids outside [0, n_actions) would alias other ids in the 8-bit field
static int check_next_ids_host(const prl_buf *b, int64_t n, const int32_t *next_action) {
    if (!next_action) return PRL_OK;
    for (int64_t i = 0; i < n; i++)
        PRL_REQUIRE(next_action[i] >= 0 && next_action[i] < b->desc.n_actions, "next action %d of transition %lld outside [0, %d)",
                    next_action[i], (long long)i, b->desc.n_actions);
    return PRL_OK;
}

static int push_host(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward, const float *next_state,
                     const uint8_t *terminated, const uint8_t *truncated, const uint8_t *next_avail_ids,
                     const int32_t *next_avail_cnt, const int32_t *next_action, const float *cost, void *stream_) {
    int rc = check_push_args(b, n, state, action, reward, terminated, truncated, next_avail_ids,
                             next_avail_cnt, next_action, cost);
    if (rc || n == 0) return rc;
    rc = check_next_ids_host(b, n, next_action);
    if (rc) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    rc = ensure_staging(b);
    if (rc) return rc;
    const int W = b->lay.record_words;
    const int64_t C = b->desc.capacity;
    // only the last `capacity` transitions of an oversized push can survive
    int64_t skip = n > C ? n - C : 0;
    if (skip) {
        b->write_pos = (b->write_pos + skip) % C;
        b->len = C;
    }
    for (int64_t i0 = skip; i0 < n;) {
        int64_t m = n - i0;
        if (m > b->stage_records) m = b->stage_records;
        if (m > C - b->write_pos) m = C - b->write_pos;  // contiguous run up to the ring end
        const int sb = b->stage_next;
        b->stage_next ^= 1;
        PRL_CUDA(cudaEventSynchronize(b->stage_done[sb]));
        uint32_t *st = b->stage[sb];
        pack_records_host(b, st, i0, m, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt,
                          next_action, cost);
        PRL_CUDA(cudaMemcpyAsync(b->records + b->write_pos * W, st, m * (int64_t)W * 4,
                                 cudaMemcpyHostToDevice, stream));
        PRL_CUDA(cudaEventRecord(b->stage_done[sb], stream));
        b->write_pos = (b->write_pos + m) % C;
        b->len = b->len + m > C ? C : b->len + m;
        i0 += m;
    }
    return PRL_OK;
}

extern "C" int prl_buf_push_host(prl_buf *b, int64_t n, const float *state, const void *action,
                                 const float *reward, const float *next_state,
                                 const uint8_t *terminated, const uint8_t *truncated,
                                 const uint8_t *next_avail_ids, const int32_t *next_avail_cnt,
                                 void *stream_) {
    return push_host(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, nullptr,
                     nullptr, stream_);
}

extern "C" int prl_buf_push_host_cost(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward,
                                      const float *next_state, const uint8_t *terminated, const uint8_t *truncated,
                                      const uint8_t *next_avail_ids, const int32_t *next_avail_cnt, const float *cost, void *stream_) {
    PRL_REQUIRE(cost || n == 0, "null cost");
    return push_host(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, nullptr,
                     cost, stream_);
}

extern "C" int prl_buf_push_host_sarsa(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward,
                                       const float *next_state, const uint8_t *terminated, const uint8_t *truncated,
                                       const uint8_t *next_avail_ids, const int32_t *next_avail_cnt, const int32_t *next_action,
                                       void *stream_) {
    PRL_REQUIRE(next_action || n == 0, "null next_action");
    return push_host(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, next_action,
                     nullptr, stream_);
}

// The same push for `count` buffers of one layout at once (a vectorised environment feeding a learner group):
// sources are [count][n][...] host arrays.  Records are packed by a few worker threads (pure CPU work), the copies are
// enqueued by the calling thread.  Buffers whose push would wrap the ring or exceed the staging area take the
// single-buffer path.
static int push_host_multi(prl_buf *const *bufs, int count, int64_t n, const float *state, const void *action, const float *reward,
                           const float *next_state, const uint8_t *terminated, const uint8_t *truncated, const int32_t *next_action,
                           void *stream_) {
    PRL_REQUIRE(bufs && count > 0, "null / empty buffer list");
    PRL_REQUIRE(n >= 0, "negative count");
    for (int i = 0; i < count; i++) {
        int rc = check_next_action(bufs[i], next_action);
        if (rc) return rc;
        // no cost argument here: a cost buffer is refused rather than given cost 0
        rc = check_cost(bufs[i], nullptr);
        if (rc) return rc;
    }
    if (n == 0) return PRL_OK;
    PRL_REQUIRE(state && action && reward && terminated && truncated, "null field array");
    if (next_action)
        for (int i = 0; i < count; i++) {
            int rc = check_next_ids_host(bufs[i], n, next_action + (size_t)i * n);
            if (rc) return rc;
        }
    cudaStream_t stream = (cudaStream_t)stream_;
    struct Job { prl_buf *b; uint32_t *st; int sb; int idx; };
    std::vector<Job> fast;
    std::vector<int> slow;
    for (int i = 0; i < count; i++) {
        prl_buf *b = bufs[i];
        PRL_REQUIRE(b, "null buffer %d", i);
        PRL_REQUIRE(b->lay.record_words == bufs[0]->lay.record_words && b->desc.obs_dim == bufs[0]->desc.obs_dim &&
                        b->desc.flags == bufs[0]->desc.flags && b->lay.act_words == bufs[0]->lay.act_words,
                    "buffers of one multi-push must share one record layout");
        int rc = ensure_staging(b);
        if (rc) return rc;
        if (n <= b->stage_records && n <= b->desc.capacity - b->write_pos) {
            const int sb = b->stage_next;
            b->stage_next ^= 1;
            PRL_CUDA(cudaEventSynchronize(b->stage_done[sb]));
            fast.push_back(Job{b, b->stage[sb], sb, i});
        } else {
            slow.push_back(i);
        }
    }
    const int obs = bufs[0]->desc.obs_dim, aw = bufs[0]->lay.act_words;
    auto src = [&](int i, const float *&s, const void *&a, const float *&r, const float *&ns, const uint8_t *&te, const uint8_t *&tr,
                   const int32_t *&na) {
        s = state + (size_t)i * n * obs;
        a = (bufs[0]->desc.flags & PRL_BUF_DISCRETE) ? (const void *)((const int32_t *)action + (size_t)i * n)
                                                     : (const void *)((const float *)action + (size_t)i * n * aw);
        r = reward + (size_t)i * n;
        ns = next_state ? next_state + (size_t)i * n * obs : nullptr;
        te = terminated + (size_t)i * n;
        tr = truncated + (size_t)i * n;
        na = next_action ? next_action + (size_t)i * n : nullptr;
    };
    const int T = (int)std::min<size_t>(8, fast.size());
    auto work = [&](int t) {
        for (size_t j = t; j < fast.size(); j += T) {
            const float *s, *r, *ns; const void *a; const uint8_t *te, *tr; const int32_t *na;
            src(fast[j].idx, s, a, r, ns, te, tr, na);
            pack_records_host(fast[j].b, fast[j].st, 0, n, s, a, r, ns, te, tr, nullptr, nullptr, na, nullptr);
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < T; t++) pool.emplace_back(work, t);
    if (T > 0) work(0);
    for (auto &th : pool) th.join();
    for (const Job &j : fast) {
        prl_buf *b = j.b;
        const int W = b->lay.record_words;
        const int64_t C = b->desc.capacity;
        PRL_CUDA(cudaMemcpyAsync(b->records + b->write_pos * W, j.st, n * (int64_t)W * 4, cudaMemcpyHostToDevice, stream));
        PRL_CUDA(cudaEventRecord(b->stage_done[j.sb], stream));
        b->write_pos = (b->write_pos + n) % C;
        b->len = b->len + n > C ? C : b->len + n;
    }
    for (int i : slow) {
        const float *s, *r, *ns; const void *a; const uint8_t *te, *tr; const int32_t *na;
        src(i, s, a, r, ns, te, tr, na);
        int rc = push_host(bufs[i], n, s, a, r, ns, te, tr, nullptr, nullptr, na, nullptr, stream_);
        if (rc) return rc;
    }
    return PRL_OK;
}

extern "C" int prl_buf_push_host_multi(prl_buf *const *bufs, int count, int64_t n, const float *state, const void *action,
                                       const float *reward, const float *next_state, const uint8_t *terminated,
                                       const uint8_t *truncated, void *stream_) {
    return push_host_multi(bufs, count, n, state, action, reward, next_state, terminated, truncated, nullptr, stream_);
}

extern "C" int prl_buf_push_host_multi_sarsa(prl_buf *const *bufs, int count, int64_t n, const float *state, const void *action,
                                             const float *reward, const float *next_state, const uint8_t *terminated,
                                             const uint8_t *truncated, const int32_t *next_action, void *stream_) {
    PRL_REQUIRE(next_action || n == 0, "null next_action");
    return push_host_multi(bufs, count, n, state, action, reward, next_state, terminated, truncated, next_action, stream_);
}

// K1: pack struct-of-arrays device sources into ring records; one warp per
// record, lanes stride the record's words (coalesced 128 B stores).
__global__ void k_pack_records(uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A,
                               int flags, int64_t capacity, int64_t write_pos, int64_t first,
                               int64_t n, const float *__restrict__ state,
                               const void *__restrict__ action, const float *__restrict__ reward,
                               const float *__restrict__ next_state,
                               const uint8_t *__restrict__ terminated,
                               const uint8_t *__restrict__ truncated,
                               const uint8_t *__restrict__ ids, const int32_t *__restrict__ cnts,
                               const int32_t *__restrict__ next_action, int off_cost, const float *__restrict__ cost) {
    const int lane = threadIdx.x & 31;
    const int64_t w = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    if (w >= n) return;
    const int64_t s = first + w;
    uint32_t *r = records + ((write_pos + w) % capacity) * L.record_words;
    for (int p = lane; p < L.record_words; p += 32) {
        uint32_t v = 0;
        if (p < L.off_next_state) {
            if (p < obs) v = __float_as_uint(state[s * obs + p]);
        } else if (p < L.off_action) {
            int q = p - L.off_next_state;
            if (q < obs && next_state) v = __float_as_uint(next_state[s * obs + q]);
        } else if (p < L.off_reward) {
            int q = p - L.off_action;
            v = (flags & PRL_BUF_DISCRETE) ? (uint32_t)((const int32_t *)action)[s]
                                           : __float_as_uint(((const float *)action)[s * L.act_words + q]);
        } else if (p == L.off_reward) {
            v = __float_as_uint(reward[s]);
        } else if (p == L.off_flags) {
            uint32_t c = (flags & PRL_BUF_DISCRETE) ? (uint32_t)A : 0u;
            if (cnts) c = (uint32_t)cnts[s];
            v = (terminated[s] ? 1u : 0u) | (truncated[s] ? 2u : 0u) | (c << 8) |
                (next_action ? ((uint32_t)next_action[s] & 0xffu) << 24 : 0u);
        } else if (p == off_cost) {
            v = __float_as_uint(cost[s]);
        } else if ((flags & PRL_BUF_DYNAMIC_ACTIONS) && (off_cost < 0 || p < off_cost)) {
            int a0 = (p - L.off_avail) * 4;
            uint32_t c = cnts ? (uint32_t)cnts[s] : (uint32_t)A;
            for (int j = 0; j < 4; j++) {
                int a = a0 + j;
                uint32_t id = 0;
                if (a < A && (uint32_t)a < c) id = ids ? ids[s * A + a] : (uint32_t)a;
                v |= id << (8 * j);
            }
        }
        r[p] = v;
    }
}

static int push_device(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward, const float *next_state,
                       const uint8_t *terminated, const uint8_t *truncated, const uint8_t *next_avail_ids,
                       const int32_t *next_avail_cnt, const int32_t *next_action, const float *cost, void *stream_) {
    int rc = check_push_args(b, n, state, action, reward, terminated, truncated, next_avail_ids,
                             next_avail_cnt, next_action, cost);
    if (rc || n == 0) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t C = b->desc.capacity;
    int64_t first = n > C ? n - C : 0;
    if (first) {
        b->write_pos = (b->write_pos + first) % C;
        b->len = C;
    }
    int64_t m = n - first;
    const int threads = 256;
    int64_t blocks = (m * 32 + threads - 1) / threads;
    k_pack_records<<<(unsigned)blocks, threads, 0, stream>>>(
        b->records, b->lay, b->desc.obs_dim, b->desc.n_actions, b->desc.flags, C, b->write_pos, first,
        m, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, next_action,
        cost_word(&b->desc), cost);
    PRL_CUDA(cudaGetLastError());
    b->write_pos = (b->write_pos + m) % C;
    b->len = b->len + m > C ? C : b->len + m;
    return PRL_OK;
}

extern "C" int prl_buf_push_device(prl_buf *b, int64_t n, const float *state, const void *action,
                                   const float *reward, const float *next_state,
                                   const uint8_t *terminated, const uint8_t *truncated,
                                   const uint8_t *next_avail_ids, const int32_t *next_avail_cnt,
                                   void *stream_) {
    return push_device(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, nullptr,
                       nullptr, stream_);
}

extern "C" int prl_buf_push_device_cost(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward,
                                        const float *next_state, const uint8_t *terminated, const uint8_t *truncated,
                                        const uint8_t *next_avail_ids, const int32_t *next_avail_cnt, const float *cost,
                                        void *stream_) {
    PRL_REQUIRE(cost || n == 0, "null cost");
    return push_device(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, nullptr,
                       cost, stream_);
}

extern "C" int prl_buf_push_device_sarsa(prl_buf *b, int64_t n, const float *state, const void *action, const float *reward,
                                         const float *next_state, const uint8_t *terminated, const uint8_t *truncated,
                                         const uint8_t *next_avail_ids, const int32_t *next_avail_cnt, const int32_t *next_action,
                                         void *stream_) {
    PRL_REQUIRE(next_action || n == 0, "null next_action");
    return push_device(b, n, state, action, reward, next_state, terminated, truncated, next_avail_ids, next_avail_cnt, next_action,
                       nullptr, stream_);
}

// Shard of a logical replay buffer of `world * capacity` transitions (SURVEY.md 8e): the transition with global
// write counter g lives on rank g mod world at local slot (g div world) mod capacity.  `global_pushed` = pushes to
// the logical buffer so far; the local content must be exactly this rank's share, pushed in order.
extern "C" int prl_buf_set_shard(prl_buf *b, int rank, int world, int64_t global_pushed) {
    PRL_REQUIRE(b, "null buffer");
    PRL_REQUIRE(world >= 1 && world <= 16 && rank >= 0 && rank < world && global_pushed >= 0, "bad shard description");
    PRL_REQUIRE(world == 1 || !(b->desc.flags & PRL_BUF_COST), "a buffer with costs (PRL_BUF_COST) cannot be sharded");
    const int64_t mine = global_pushed / world + ((global_pushed % world) > rank ? 1 : 0);   // g < global_pushed, g mod world == rank
    const int64_t expect = mine < b->desc.capacity ? mine : b->desc.capacity;
    PRL_REQUIRE(world == 1 || b->len == expect,
                "shard holds %lld transitions, %lld expected for rank %d of %d after %lld global pushes", (long long)b->len,
                (long long)expect, rank, world, (long long)global_pushed);
    PRL_REQUIRE(world == 1 || b->write_pos == mine % b->desc.capacity, "shard ring position does not match the global write counter");
    b->shard_rank = rank; b->shard_world = world; b->g_pushed = global_pushed;
    return PRL_OK;
}
// population of the logical buffer a shard belongs to (= prl_buf_len for an unsharded buffer)
extern "C" int64_t prl_buf_global_len(const prl_buf *b) {
    if (!b) return 0;
    if (b->shard_world <= 1) return b->len;
    const int64_t cap = b->desc.capacity * b->shard_world;
    return b->g_pushed < cap ? b->g_pushed : cap;
}

// --------------------------------------------------------------------------
// RNG state hand-off
// --------------------------------------------------------------------------
extern "C" int prl_rng_set_state(prl_buf *b, const uint32_t *st, void *stream) {
    PRL_REQUIRE(b && st, "null argument");
    PRL_REQUIRE(st[624] <= 624, "MT19937 position must be in [0,624]");
    uint32_t any = 0;
    for (int i = 0; i < 624; i++) any |= st[i];
    PRL_REQUIRE(any != 0, "all-zero MT19937 state (not a state random.getstate() can return; it never leaves zero)");
    PRL_CUDA(cudaMemcpyAsync(b->mt_state, st, 625 * 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    PRL_CUDA(cudaStreamSynchronize((cudaStream_t)stream));  // `st` may be a temporary
    return PRL_OK;
}
extern "C" int prl_rng_get_state(prl_buf *b, uint32_t *st, void *stream) {
    PRL_REQUIRE(b && st, "null argument");
    PRL_CUDA(cudaMemcpyAsync(st, b->mt_state, 625 * 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    PRL_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return PRL_OK;
}
// CPython init_by_array (Modules/_randommodule.c), done on the host: 624 words.
extern "C" int prl_rng_seed(prl_buf *b, const uint32_t *key, int key_len, void *stream) {
    PRL_REQUIRE(b && key && key_len > 0, "bad key");
    uint32_t st[625];
    st[0] = 19650218u;
    for (int i = 1; i < 624; i++) st[i] = 1812433253u * (st[i - 1] ^ (st[i - 1] >> 30)) + (uint32_t)i;
    int i = 1, j = 0;
    for (int k = (624 > key_len ? 624 : key_len); k; k--) {
        st[i] = (st[i] ^ ((st[i - 1] ^ (st[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
        i++, j++;
        if (i >= 624) { st[0] = st[623]; i = 1; }
        if (j >= key_len) j = 0;
    }
    for (int k = 623; k; k--) {
        st[i] = (st[i] ^ ((st[i - 1] ^ (st[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
        i++;
        if (i >= 624) { st[0] = st[623]; i = 1; }
    }
    st[0] = 0x80000000u;
    st[624] = 624;
    return prl_rng_set_state(b, st, stream);
}

// --------------------------------------------------------------------------
// K2: MT19937-exact sampler, stand-alone kernel (device routines in sampler.cuh)
// --------------------------------------------------------------------------
__global__ void __launch_bounds__(kSamplerThreads, 1)
k_sample_indices(uint32_t *__restrict__ mt_state, SamplerParams p, int rounds) {
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ SamplerState S;
    sampler_init(S, mt_state, dyn, p);
    sampler_advance(S, dyn, p, rounds);
    __syncthreads();
    sampler_store(S, mt_state);
}

static int64_t sample_setsize(int64_t k) {  // Lib/random.py:432-434
    int64_t s = 21;
    if (k > 5) { int64_t p = 1; while (p < 3 * k) p *= 4; s += p; }
    return s;
}

// sampler geometry for `k` draws from the buffer's current population (shared with
// the fused learner kernels); returns the dynamic shared memory the sampler needs
int prl_sampler_params(const prl_buf *b, int k, prl::SamplerParams *sp, size_t *smem_bytes) {
    const bool shard = b->shard_world > 1;
    const int64_t n = prl_buf_global_len(b);   // a shard draws from the LOGICAL buffer: every rank the same indices
    if (k > n)
        return fail(PRL_EINVAL, "Can't get a batch of size %d from a replay buffer with only %lld elements", k,
                    (long long)n);
    sp->n = (uint32_t)n; sp->k = k;
    sp->use_pool = n <= sample_setsize(k);
    sp->table_cap = 0;
    if (sp->use_pool) {
        *smem_bytes = (size_t)n * 4;
    } else {
        uint32_t cap = 64;
        while (cap < (uint32_t)(2 * k)) cap <<= 1;
        // a sparser table (load <= 1/8 while it stays under 32 KB) keeps the probe sequences of a 32-lane chunk short
        for (int g = 0; g < 2 && (size_t)cap * 2 * 8 <= 32 * 1024; g++) cap <<= 1;
        sp->table_cap = cap;
        *smem_bytes = (size_t)cap * 8;
    }
    if (*smem_bytes > 200 * 1024) return fail(PRL_EUNSUPPORTED, "sample size %d too large for the on-chip sampler", k);
    sp->head = shard ? 0 : prl_buf_head(b);     // sharded: out_slot carries the logical index, owners map it themselves
    sp->capacity = shard ? b->desc.capacity * b->shard_world : b->desc.capacity;
    sp->out_logical = nullptr; sp->out_slot = nullptr;
    return PRL_OK;
}

extern "C" int prl_buf_sample_indices(prl_buf *b, int rounds, int k, int32_t *out_logical,
                                      int32_t *out_slot, void *stream_) {
    PRL_REQUIRE(b, "null buffer");
    PRL_REQUIRE(rounds >= 0 && k >= 0, "negative rounds / k");
    SamplerParams sp;
    size_t smem = 0;
    int rc = prl_sampler_params(b, k, &sp, &smem);
    if (rc) return rc;
    if (rounds == 0 || k == 0) return PRL_OK;
    sp.out_logical = out_logical;
    sp.out_slot = out_slot;
    PRL_CUDA(cudaFuncSetAttribute(k_sample_indices, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    k_sample_indices<<<1, kSamplerThreads, smem, (cudaStream_t)stream_>>>(b->mt_state, sp, rounds);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// --------------------------------------------------------------------------
// gather into TransitionBatch field layout; one warp per sampled record
// --------------------------------------------------------------------------
__global__ void k_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int flags,
                         const int32_t *__restrict__ slots, int k, float *__restrict__ state,
                         void *__restrict__ action, float *__restrict__ reward,
                         float *__restrict__ next_state, uint8_t *__restrict__ terminated,
                         uint8_t *__restrict__ truncated, float *__restrict__ next_avail,
                         uint8_t *__restrict__ next_mask) {
    const int lane = threadIdx.x & 31;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= k) return;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        if (state) state[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        if (next_state) next_state[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    const uint32_t fl = r[L.off_flags];
    if (lane == 0) {
        if (reward) reward[w] = __uint_as_float(r[L.off_reward]);
        if (terminated) terminated[w] = fl & 1u;
        if (truncated) truncated[w] = (fl >> 1) & 1u;
    }
    if (action) {
        if (flags & PRL_BUF_DISCRETE) {
            if (lane == 0) ((long long *)action)[w] = (long long)(int32_t)r[L.off_action];
        } else {
            for (int p = lane; p < L.act_words; p += 32)
                ((float *)action)[(size_t)w * L.act_words + p] = __uint_as_float(r[L.off_action + p]);
        }
    }
    if ((flags & PRL_BUF_DISCRETE) && (next_avail || next_mask)) {
        const uint32_t cnt = (fl >> 8) & 0xffffu;
        const uint8_t *ids = (const uint8_t *)(r + L.off_avail);
        for (int a = lane; a < A; a += 32) {
            const bool avail = (uint32_t)a < cnt;
            float id = 0.f;
            if (avail) id = (flags & PRL_BUF_DYNAMIC_ACTIONS) ? (float)ids[a] : (float)a;
            if (next_avail) next_avail[(size_t)w * A + a] = id;
            if (next_mask) next_mask[(size_t)w * A + a] = avail ? 0 : 1;
        }
    }
}

extern "C" int prl_buf_gather(const prl_buf *b, const int32_t *slot_dev, int k, float *state, void *action,
                              float *reward, float *next_state, uint8_t *terminated, uint8_t *truncated,
                              float *next_avail, uint8_t *next_unavail_mask, void *stream_) {
    PRL_REQUIRE(b && slot_dev, "null argument");
    if (k <= 0) return PRL_OK;
    const int threads = 256;
    const int blocks = (k * 32 + threads - 1) / threads;
    k_gather<<<blocks, threads, 0, (cudaStream_t)stream_>>>(b->records, b->lay, b->desc.obs_dim,
                                                            b->desc.n_actions, b->desc.flags, slot_dev, k,
                                                            state, action, reward, next_state, terminated,
                                                            truncated, next_avail, next_unavail_mask);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// the committed next action of k records (PRL_BUF_NEXT_ACTION): bits 24..31 of the flags word, as int64 ids
__global__ void k_gather_next_action(const uint32_t *__restrict__ records, prl_buf_layout L, const int32_t *__restrict__ slots, int k,
                                     long long *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    out[i] = (long long)(records[(size_t)slots[i] * L.record_words + L.off_flags] >> 24);
}

extern "C" int prl_buf_gather_next_action(const prl_buf *b, const int32_t *slot_dev, int k, int64_t *out_dev, void *stream_) {
    PRL_REQUIRE(b && slot_dev && out_dev, "null argument");
    PRL_REQUIRE(b->desc.flags & PRL_BUF_NEXT_ACTION, "the buffer was created without PRL_BUF_NEXT_ACTION: it stores no next action");
    if (k <= 0) return PRL_OK;
    k_gather_next_action<<<(k + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(b->records, b->lay, slot_dev, k, (long long *)out_dev);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// the cost word of k records (PRL_BUF_COST)
__global__ void k_gather_cost(const uint32_t *__restrict__ records, int W, int off_cost, const int32_t *__restrict__ slots, int k,
                              float *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    out[i] = __uint_as_float(records[(size_t)slots[i] * W + off_cost]);
}

extern "C" int prl_buf_gather_cost(const prl_buf *b, const int32_t *slot_dev, int k, float *out_dev, void *stream_) {
    PRL_REQUIRE(b && slot_dev && out_dev, "null argument");
    PRL_REQUIRE(b->desc.flags & PRL_BUF_COST, "the buffer was created without PRL_BUF_COST: it stores no cost");
    if (k <= 0) return PRL_OK;
    k_gather_cost<<<(k + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(b->records, b->lay.record_words, cost_word(&b->desc), slot_dev, k,
                                                                      out_dev);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
