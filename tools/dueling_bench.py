"""Developer tool: rates of the dueling DQN learner (pearl_b200.B200DeepQLearning / B200DoubleDQN with
network_type=DuelingQValueNetwork) on one GPU, next to the eager-torch restatement (oracle/dueling_oracle.py) on the host:
  DuelingDQN_method  the shape of Pearl's DuelingDQN_method benchmark (DeepQLearning, obs 4, 2 actions, [64, 64],
                     batch 32): gradient-steps/s of learn()
  stress_dqn         DeepQLearning, obs 128, 16 actions, [256, 256], batch 256, dynamic next-action sets:
                     gradient-steps/s of learn()
  stress_ddqn        the same shape with DoubleDQN
  *_batch            the same shapes through learn_batch() (PearlAgent.learn_batch's path): calls/s, each call one round
                     on a batch already on the device (every action current), with the read-back of its loss
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up; the launches
per round are the library's count.  Prints the card's name and power limit with the numbers.

    python tools/dueling_bench.py [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pearl_b200  # noqa: E402
from oracle.dueling_oracle import OracleDueling, one_hot_batch  # noqa: E402

SHAPES = {"DuelingDQN_method": dict(obs=4, A=2, hidden=64, B=32, n=100_000, dynamic=False, double=False),
          "stress_dqn": dict(obs=128, A=16, hidden=256, B=256, n=200_000, dynamic=True, double=False),
          "stress_ddqn": dict(obs=128, A=16, hidden=256, B=256, n=200_000, dynamic=True, double=True)}


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


def learner(shape, rounds):
    h, A = shape["hidden"], shape["A"]
    cls = pearl_b200.B200DoubleDQN if shape["double"] else pearl_b200.B200DeepQLearning
    torch.manual_seed(3)
    return cls(state_dim=shape["obs"], action_space=Space(A), hidden_dims=[h, h], training_rounds=rounds, batch_size=shape["B"],
               network_type=pearl_b200.DuelingQValueNetwork, action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda:0")


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


def gpu_rates(name, shape, d, rounds_per_call=200):
    n, t = shape["n"], torch.from_numpy
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    extra = dict(next_available_ids=t(d["next_ids"]), next_available_count=t(d["next_count"])) if shape["dynamic"] else {}
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=shape["A"], **extra)
    buf.seed(1)
    pl = learner(shape, rounds_per_call)
    rep = pl.learn(buf, trace=True)                             # warm-up: capture, module loads, algorithm choice
    out = {name: dict(launches_per_round=rep["launches"] / rounds_per_call)}
    rate, win = timed(lambda: pl.learn(buf), rounds_per_call)
    out[name].update(steps_per_s=rate, window_s=win)
    rng = np.random.Generator(np.random.PCG64(7))
    batches = [batch_of(shape, d, rng.choice(n, size=shape["B"], replace=False), "cuda") for _ in range(64)]
    k = [0]

    def one():
        pl.learn_batch(batches[k[0] % len(batches)])
        k[0] += 1
    for _ in range(8):
        one()                                               # warm-up of the learn_batch graph
    rate, win = timed(one, 1)
    out[f"{name}_batch"] = dict(calls_per_s=rate, window_s=win)
    return out


def host_rate(shape, d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    h, A = shape["hidden"], shape["A"]
    orc = OracleDueling(shape["obs"], A, (h, h), double=shape["double"])
    rng = np.random.Generator(np.random.PCG64(5))
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or steps < 3:
        i = rng.choice(shape["n"], size=shape["B"], replace=False)
        b = one_hot_batch(A, *(torch.from_numpy(d[k][i]) for k in ("state", "action", "reward", "next_state", "term")), None,
                          d["next_ids"][i].astype(np.int64), d["next_count"][i])
        orc.training_steps += 1
        orc.learn_batch(b)
        steps += 1
    dt = time.perf_counter() - t0
    return dict(steps_per_s=steps / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for dueling_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(shape)
        hst = host_rate(shape, d)
        for k, g in gpu_rates(name, shape, d).items():
            res["shapes"][k] = dict(shape=shape, gpu=g, host_oracle=hst)
            rate = (f"{g['steps_per_s']:.0f} gradient-steps/s ({g['launches_per_round']:.0f} launches/round)" if "steps_per_s" in g
                    else f"{g['calls_per_s']:.0f} learn_batch calls/s")
            print(f"{k}: GPU {rate} over {g['window_s']:.1f} s; host eager-torch oracle {hst['steps_per_s']:.1f} steps/s "
                  f"({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dueling_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
