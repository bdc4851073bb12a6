"""Developer tool: rates of the multi-head DQN learner (pearl_b200.B200DeepQLearning / B200DoubleDQN with
network_type=VanillaQValueMultiHeadNetwork, plain or conservative) on one GPU, next to the one-hot B200DeepQLearning
(VanillaQValueNetwork, engine "simt") at the same shape in the same run:
  integration  the shape of Pearl's multi-head integration test (obs 4, 2 actions, [64, 64], batch 128)
  stress       obs 128, 16 actions, [256, 256], batch 256, dynamic next-action sets
each for dqn, ddqn and cql_dqn (conservative DeepQLearning, alpha 2): gradient-steps/s of learn() over a B200ReplayBuffer,
and learn_batch() calls/s (PearlAgent.learn_batch's path: one round on a batch already on the device, every action
current, with the read-back of its loss).  onehot_dqn is the one-hot learner's learn().
The rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up call; the launches
per round are the library's count.  Prints the card's name and power limit with the numbers.  --profile adds a
torch.profiler table of the GPU time per kernel of one stress-shape round (graphs off) for the multi-head and the one-hot
DQN learner.

    python tools/multihead_bench.py [--out DIR] [--profile]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pearl_b200  # noqa: E402

SHAPES = {"integration": dict(obs=4, A=2, hidden=64, B=128, n=100_000, dynamic=False),
          "stress": dict(obs=128, A=16, hidden=256, B=256, n=200_000, dynamic=True)}
VARIANTS = {"dqn": dict(double=False, alpha=None), "ddqn": dict(double=True, alpha=None), "cql_dqn": dict(double=False, alpha=2.0)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(shape, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    n, obs, A = shape["n"], shape["obs"], shape["A"]
    d = dict(state=rng.standard_normal((n, obs), dtype=np.float32), next_state=rng.standard_normal((n, obs), dtype=np.float32),
             reward=rng.standard_normal(n, dtype=np.float32), term=rng.random(n) < 0.01, action=rng.integers(0, A, size=n).astype(np.int32))
    cnt = rng.integers(1, A + 1, size=n).astype(np.int32) if shape["dynamic"] else np.full(n, A, np.int32)
    ids = np.argsort(rng.random((n, A)), axis=1)           # a random order of every action; the first cnt are available
    d.update(next_ids=ids.astype(np.uint8), next_count=cnt)
    return d


class Space:
    def __init__(self, A):
        self.n, self.actions, self.actions_batch = A, [torch.tensor([i]) for i in range(A)], torch.arange(A).view(A, 1)


def learner(shape, rounds, double=False, alpha=None, multihead=True):
    h, A = shape["hidden"], shape["A"]
    cls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    kw = dict(network_type=pearl_b200.VanillaQValueMultiHeadNetwork) if multihead else dict(engine="simt")
    if alpha is not None:
        kw.update(is_conservative=True, conservative_alpha=alpha)
    torch.manual_seed(3)
    return cls(state_dim=shape["obs"], action_space=Space(A), hidden_dims=[h, h], training_rounds=rounds, batch_size=shape["B"],
               action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A), **kw).to("cuda:0")


def timed(fn, per_call, window_s=2.0):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    done, ms = 0, 0.0
    while ms < window_s * 1e3:
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        done += per_call
    return done / (ms / 1e3), ms / 1e3


def batch_of(shape, d, i, device=None):
    A = shape["A"]
    t = lambda k: torch.from_numpy(d[k][i]).to(device)  # noqa: E731
    mask = torch.arange(A, device=device).view(1, A) >= t("next_count").view(-1, 1)
    curr = torch.arange(A, device=device).float().view(1, A, 1).expand(len(i), -1, -1)
    return pearl_b200.TransitionBatch(state=t("state"), action=t("action").long().view(-1, 1), reward=t("reward"),
                                      next_state=t("next_state"), terminated=t("term"), curr_available_actions=curr,
                                      next_available_actions=t("next_ids").float().view(len(i), A, 1),
                                      next_unavailable_actions_mask=mask)


def make_buffer(shape, d):
    n, t = shape["n"], torch.from_numpy
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    extra = dict(next_available_ids=t(d["next_ids"]), next_available_count=t(d["next_count"])) if shape["dynamic"] else {}
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=shape["A"], **extra)
    buf.seed(1)
    return buf


def gpu_rates(shape, d, buf, pl, rounds_per_call, batch=True):
    rep = pl.learn(buf, trace=True)                             # warm-up: capture, module loads, algorithm choice
    out = dict(launches_per_round=rep["launches"] / rounds_per_call) if "launches" in rep else {}
    out["steps_per_s"], out["window_s"] = timed(lambda: pl.learn(buf), rounds_per_call)
    if batch:
        rng = np.random.Generator(np.random.PCG64(7))
        batches = [batch_of(shape, d, rng.choice(shape["n"], size=shape["B"], replace=False), "cuda") for _ in range(64)]
        k = [0]

        def one():
            pl.learn_batch(batches[k[0] % len(batches)])
            k[0] += 1
        for _ in range(8):
            one()                                               # warm-up of the learn_batch graph
        out["batch_calls_per_s"], out["batch_window_s"] = timed(one, 1)
    return out


def profile_round(shape, d, buf, multihead):
    """GPU time per kernel name of a few learn() rounds with plain launches (torch.profiler)."""
    pl = learner(shape, 1, multihead=multihead)
    if multihead:
        pl.use_cuda_graph = False
    pl.learn(buf)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    rounds = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            pl.learn(buf)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0 and e.count > 0:
            rows[e.key[:110]] = dict(us_per_round=t / rounds, launches_per_round=e.count / rounds)
    return dict(sorted(rows.items(), key=lambda kv: -kv[1]["us_per_round"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for multihead_bench.json")
    ap.add_argument("--profile", action="store_true", help="kernel table of one stress-shape round, multi-head and one-hot")
    args = ap.parse_args()
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(shape)
        buf = make_buffer(shape, d)
        rpc = 200
        for v, kw in VARIANTS.items():
            g = gpu_rates(shape, d, buf, learner(shape, rpc, **kw), rpc)
            res["shapes"][f"{name}_{v}"] = dict(shape=shape, gpu=g)
            print(f"{name}_{v}: learn() {g['steps_per_s']:.0f} gradient-steps/s ({g['launches_per_round']:.0f} launches/round); "
                  f"learn_batch() {g['batch_calls_per_s']:.0f} calls/s")
        g = gpu_rates(shape, d, buf, learner(shape, rpc, multihead=False), rpc, batch=False)
        res["shapes"][f"{name}_onehot_dqn"] = dict(shape=shape, gpu=g)
        print(f"{name}_onehot_dqn: learn() {g['steps_per_s']:.0f} gradient-steps/s (one persistent kernel per call)")
        if args.profile and name == "stress":
            for mh in (True, False):
                tab = profile_round(shape, d, buf, mh)
                res[f"profile_{'multihead' if mh else 'onehot'}"] = tab
                print(f"per-round GPU time, {'multi-head' if mh else 'one-hot'} DQN (plain launches):")
                for k, r in list(tab.items())[:14]:
                    print(f"  {r['us_per_round']:8.2f} us  x{r['launches_per_round']:.0f}  {k}")
                print(f"  total {sum(r['us_per_round'] for r in tab.values()):.2f} us")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "multihead_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
