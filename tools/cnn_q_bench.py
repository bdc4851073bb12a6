"""Developer tool: rates of the CNN DQN learner (pearl_b200.B200DeepQLearning / B200DoubleDQN with CNNQValueNetwork or
CNNQValueMultiHeadNetwork) on one GPU at the shape of Pearl's Atari benchmark (PongNoFrameskip-v4: 4 x 84 x 84 stacked
frames, conv 8/4/3 with 32/64/64 channels and strides 4/2/1, FC 512, 6 actions, batch 32) over a 50 000-transition
B200ReplayBuffer (about 11.3 GB of ring):
  gradient-steps/s of learn(), and learn_batch() calls/s (one round on a batch already on the device, with the read-back
  of its loss), for dqn, ddqn, mh_dqn and mh_ddqn; the launches per round (the library's count); the algorithmic FLOP of
  one round computed from the shapes below; and the same round of the eager-torch oracle (oracle/cnn_q_oracle.py) on the
  host, timed in the same run.
GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up call.  Prints the
card's name, power limit and SM clock read in the same run.

    python tools/cnn_q_bench.py [--out DIR] [--n 50000]
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
from oracle import cnn_q_oracle as orc  # noqa: E402

PONG = dict(input=(4, 84, 84), conv=[(32, 8, 4, 0), (64, 4, 2, 0), (64, 3, 1, 0)], hidden=[512], n_actions=6)
B = 32
VARIANTS = {"dqn": (False, False), "ddqn": (False, True), "mh_dqn": (True, False), "mh_ddqn": (True, True)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def flop_per_round(spec, double) -> float:
    """2 x multiply-adds of the products one round needs: the target net on B next states, the online net on B states
    (DoubleDQN: and on B next states), every action's FC values for the next states (vanilla: the layer-0 feature
    product once per state, the rest per action), and the backward pass (weight and data gradients of every layer below
    the head, no data gradient into the pixels)."""
    convs, F = orc.conv_shapes(spec)
    A, hid = spec["n_actions"], spec["hidden"]
    conv = [(oc * ho * wo, c * k * k) for (c, _, _, oc, ho, wo), (_, k, _, _) in zip(convs, spec["conv"])]
    trunk = sum(m * k for m, k in conv)                                # multiply-adds per image
    dims = [F] + hid + [A if spec["multi"] else 1]
    fc_layers = [dims[i] * dims[i + 1] for i in range(len(dims) - 1)]
    if spec["multi"]:
        fc_state, fc_all = sum(fc_layers), sum(fc_layers)
    else:
        fc_state = sum(fc_layers)
        fc_all = fc_layers[0] + A * sum(fc_layers[1:])
    fwd = B * (trunk + fc_all) + B * (trunk + fc_state) + (B * (trunk + fc_all) if double else 0)
    bwd = B * (2 * sum(fc_layers) + trunk + sum(m * k for m, k in conv[1:]))
    return 2.0 * (fwd + bwd)


class Space:
    def __init__(self, A):
        self.n, self.actions, self.actions_batch = A, [torch.tensor([i]) for i in range(A)], torch.arange(A).view(A, 1)


def learner(multi, double, rounds):
    spec = PONG
    C, H, W = spec["input"]
    A = spec["n_actions"]
    cls = pearl_b200.CNNQValueMultiHeadNetwork if multi else pearl_b200.CNNQValueNetwork
    net = cls(input_width=W, input_height=H, input_channels_count=C, kernel_sizes=[8, 4, 3], output_channels_list=[32, 64, 64],
              strides=[4, 2, 1], paddings=[0, 0, 0], action_dim=A, hidden_dims_fully_connected=[512], output_dim=A if multi else 1)
    lcls = pearl_b200.B200DoubleDQN if double else pearl_b200.B200DeepQLearning
    return lcls(state_dim=C * H * W, action_space=Space(A), hidden_dims=[512], network_instance=net, learning_rate=1e-4,
                training_rounds=rounds, batch_size=B, target_update_freq=10, soft_update_tau=1.0,
                action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda:0")


def timed(fn, min_s=2.0):
    """Calls per second of fn over a window of at least min_s seconds (CUDA events around whole calls)."""
    fn()
    torch.cuda.synchronize()
    calls, total = 0, 0.0
    while total < min_s:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1) / 1e3
        calls += 5
    return calls / total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--rounds", type=int, default=50)
    args = ap.parse_args()
    torch.manual_seed(0)
    spec0 = dict(PONG, multi=False)
    n, C, H, W = args.n, *PONG["input"]
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    g = torch.Generator().manual_seed(0)
    chunk = 1000
    for i0 in range(0, n, chunk):
        m = min(chunk, n - i0)
        buf.push_batch(torch.randint(0, 256, (m, C, H, W), generator=g).float(), torch.randint(0, 6, (m,), generator=g).int(),
                       torch.randn(m, generator=g), torch.randint(0, 256, (m, C, H, W), generator=g).float(),
                       torch.rand(m, generator=g) < 0.01, torch.zeros(m, dtype=torch.bool), max_number_actions=6)
    dev = torch.device("cuda:0")
    batch = pearl_b200.TransitionBatch(
        state=torch.randint(0, 256, (B, C, H, W), device=dev).float(), action=torch.randint(0, 6, (B,), device=dev),
        reward=torch.randn(B, device=dev), terminated=torch.zeros(B, dtype=torch.bool, device=dev),
        next_state=torch.randint(0, 256, (B, C, H, W), device=dev).float())
    out = dict(card=card(), shape="Pong 4x84x84, conv 8/4/3 32/64/64 s4/2/1, FC 512, A 6, batch 32", ring_transitions=n,
               ring_gb=round(n * buf.record_bytes / 1e9, 2), params=orc.param_count(spec0), results={})
    for name, (multi, double) in VARIANTS.items():
        spec = dict(PONG, multi=multi)
        pl = learner(multi, double, args.rounds)
        learn_calls = timed(lambda: pl.learn(buf))
        launches = pl.launch_info()["launches"] // args.rounds
        pl1 = learner(multi, double, 1)
        lb = timed(lambda: pl1.learn_batch(batch))
        fl = flop_per_round(spec, double)
        steps = learn_calls * args.rounds
        # the eager-torch oracle on the host: one round on the same shape
        cpu_b = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in orc.batch_of(dict(
            state=np.random.randint(0, 256, (B, C, H, W)).astype(np.float32), next_state=np.random.randint(0, 256, (B, C, H, W)).astype(np.float32),
            action=np.random.randint(0, 6, B), reward=np.random.randn(B).astype(np.float32), terminated=np.zeros(B, bool),
            next_ids=np.tile(np.arange(6), (B, 1)), next_count=np.full(B, 6)), np.arange(B)).items()}
        w = pl.flat_parameters.cpu().clone()
        st = dict(w=w, wt=w.clone(), m=torch.zeros_like(w), v=torch.zeros_like(w), vmax=torch.zeros_like(w), step=0)
        orc.round_step(spec, st, cpu_b, double=double, gamma=0.99, tau=1.0, lr=1e-4, update_target=False)
        t0 = time.perf_counter()
        for _ in range(3):
            orc.round_step(spec, st, cpu_b, double=double, gamma=0.99, tau=1.0, lr=1e-4, update_target=False)
        host_ms = (time.perf_counter() - t0) / 3 * 1e3
        out["results"][name] = dict(learn_steps_per_s=round(steps, 1), learn_batch_calls_per_s=round(lb, 1),
                                    launches_per_round=launches, gflop_per_round=round(fl / 1e9, 3),
                                    learn_tflops=round(fl * steps / 1e12, 2), host_oracle_ms_per_round=round(host_ms, 1),
                                    host_threads=torch.get_num_threads())
        print(name, out["results"][name], flush=True)
        del pl, pl1
    print(json.dumps(out))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cnn_q_bench.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
