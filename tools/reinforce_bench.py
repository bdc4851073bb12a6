"""Developer tool: speed of the REINFORCE learner (pearl_b200.B200REINFORCE) on one GPU, next to the eager-torch restatement
(oracle/reinforce_oracle.py) on the host, at two shapes:
  REINFORCE_method  Pearl's benchmark configuration (obs 4, 2 actions, [64, 64], 8 rounds, batch 64) on a 500-transition
                    rollout (a few episodes: the agent learns after each episode and clears the buffer)
  stress            obs 128, 16 actions, [256, 256], 8 rounds, batch 256, a 20 000-transition rollout
Reported: gradient steps/s and learn() calls/s (a call = the return pass + 8 rounds), the return pass alone (critic at the
newest next_state + the serial fold) at the rollout length and at 50 000 transitions (the benchmark config's capacity),
launches per round, and the host oracle's learn() calls/s.  GPU times are CUDA events over windows of at least 2 s after a
warm-up call.  Prints the card's name and power limit with the numbers.

    python tools/reinforce_bench.py [--out DIR]
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
from pearl_b200 import _lib  # noqa: E402
from pearl_b200.replay_buffer import _stream_ptr  # noqa: E402
from oracle.reinforce_oracle import OracleREINFORCE  # noqa: E402

SHAPES = {"REINFORCE_method": dict(obs=4, A=2, hidden=64, B=64, rounds=8, n=500),
          "stress": dict(obs=128, A=16, hidden=256, B=256, rounds=8, n=20_000)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(n, obs, A, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    term = rng.random(n) < 0.01
    return dict(state=rng.standard_normal((n, obs)).astype(np.float32), next_state=rng.standard_normal((n, obs)).astype(np.float32),
                reward=(rng.standard_normal(n) * 0.1).astype(np.float32), action=rng.integers(0, A, size=n).astype(np.int32), term=term)


def make_buffer(d, A):
    n = d["state"].shape[0]
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    t = torch.from_numpy
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool),
                   max_number_actions=A)
    buf.seed(1)
    return buf


def timed(fn, window_s=2.0):
    """(calls, ms) of fn() over CUDA events, at least window_s seconds."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    calls, ms = 0, 0.0
    while ms < window_s * 1e3:
        e0.record()
        for _ in range(20):
            fn()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        calls += 20
    return calls, ms


def gpu_rate(shape, d):
    buf = make_buffer(d, shape["A"])
    h = shape["hidden"]
    pl = pearl_b200.B200REINFORCE(state_dim=shape["obs"], n_actions=shape["A"], actor_hidden_dims=[h, h], critic_hidden_dims=[h, h],
                                  training_rounds=shape["rounds"], batch_size=shape["B"], seed=3)
    trace = {}
    pl.learn(buf, trace=trace)                                  # warm-up: capture, module loads, algorithm choice
    launches = trace["launches"] / shape["rounds"]
    torch.cuda.synchronize()
    calls, ms = timed(lambda: pl.learn(buf))
    dev = pl._device

    def returns(b):
        _lib.check(pl._lib.prl_reinforce_returns(pl._handle, b.handle, _lib.ptr(pl._returns), _stream_ptr(dev)))
    rcalls, rms = timed(lambda: returns(buf), window_s=1.0)
    big = make_buffer(data(50_000, shape["obs"], shape["A"], seed=9), shape["A"])
    returns(big)
    bcalls, bms = timed(lambda: returns(big), window_s=1.0)
    return dict(steps_per_s=calls * shape["rounds"] / (ms / 1e3), learn_calls_per_s=calls / (ms / 1e3), window_s=ms / 1e3,
                launches_per_round=launches, return_pass_us=1e3 * rms / rcalls, return_pass_50k_us=1e3 * bms / bcalls)


def host_rate(shape, d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    h, B, A, n = shape["hidden"], shape["B"], shape["A"], shape["n"]
    orc = OracleREINFORCE(shape["obs"], A, (h, h), (h, h))
    rng = np.random.Generator(np.random.PCG64(5))
    calls, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or calls < 2:
        R = orc.returns(d["reward"], d["next_state"][-1], d["term"][-1])
        for _ in range(shape["rounds"]):
            i = rng.choice(n, size=min(B, n), replace=False)
            orc.learn_batch(torch.from_numpy(d["state"][i]), torch.from_numpy(d["action"][i]), R)
        calls += 1
    dt = time.perf_counter() - t0
    return dict(learn_calls_per_s=calls / dt, steps_per_s=calls * shape["rounds"] / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for reinforce_bench.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reinforce_bench needs a CUDA device")
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(shape["n"], shape["obs"], shape["A"])
        g, hst = gpu_rate(shape, d), host_rate(shape, d)
        res["shapes"][name] = dict(shape=shape, gpu=g, host_oracle=hst)
        print(f"{name}: GPU {g['steps_per_s']:.0f} gradient-steps/s, {g['learn_calls_per_s']:.0f} learn() calls/s "
              f"({g['launches_per_round']:.0f} launches/round, {g['window_s']:.1f} s); return pass {g['return_pass_us']:.1f} us "
              f"at {shape['n']} transitions, {g['return_pass_50k_us']:.1f} us at 50 000; host eager-torch oracle "
              f"{hst['learn_calls_per_s']:.2f} learn() calls/s ({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "reinforce_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
