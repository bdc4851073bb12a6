"""Developer tool: aggregate rate of the tensor-core learner group (R learners, `rounds` rounds) + phase stamps of CTA 0."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, ctypes as C
import pearl_b200
from pearl_b200 import _lib
from bench import Space, OBS, N_ACT, HIDDEN, BATCH
R = int(sys.argv[1]) if len(sys.argv) > 1 else 64
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 256
cap = int(sys.argv[3]) if len(sys.argv) > 3 else 100_000
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(1)
bufs, ls = [], []
for i in range(R):
    b = pearl_b200.B200ReplayBuffer(cap, rng="device")
    b.push_batch(torch.randn((cap, OBS), generator=g, device=dev), (torch.arange(cap, device=dev) % N_ACT).to(torch.int32),
                 torch.randn(cap, generator=g, device=dev), torch.randn((cap, OBS), generator=g, device=dev),
                 torch.rand(cap, generator=g, device=dev) < 0.02, torch.zeros(cap, dtype=torch.bool, device=dev), max_number_actions=N_ACT)
    b.seed(i + 1)
    bufs.append(b)
    ls.append(pearl_b200.B200DeepQLearning(state_dim=OBS, action_space=Space(N_ACT), hidden_dims=list(HIDDEN), training_rounds=rounds, batch_size=BATCH,
                                           action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(N_ACT),
                                           max_rounds_per_call=rounds, engine="tc").to(dev))
grp = pearl_b200.B200LearnerGroup(ls, bufs)
grp.set_kernel_timing(True)
for _ in range(2):
    grp.learn()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(3):
    grp.learn()
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / 3
print(f"R={R} rounds={rounds}: {R*rounds/dt:.4e} steps/s wall; kernel {grp.last_kernel_ms():.2f} ms -> {R*rounds/grp.last_kernel_ms()*1e3:.4e} steps/s; {grp.last_kernel_ms()*1e3/rounds:.1f} us/round")
# phase stamps (single learner launch, unchunked)
st = torch.zeros((rounds, 16), dtype=torch.int64, device=dev)
_lib.check(ls[0]._libh.prl_dqn_set_profile(ls[0]._handle, C.c_void_p(st.data_ptr())))
grp.learn()
torch.cuda.synchronize()
s = st.cpu()[4:].double()
# stamps written by k_dqn_tc: 0 round start, 1 row scalars + soft update done, 2 target tiles loaded, 3 phase T done,
# 4 online tiles + W2^T ready, 5 tile 0 layer 1 done, 6 tile 0 forward / dZ2 / dH1 done, 8 weight gradients done, 9 AdamW done
names = ["row scalars + soft upd", "load target weights", "phase T (layer 1 + all actions)", "load online weights + W2^T",
         "tile 0: online layer 1", "tile 0: fwd L2 + dZ2 + dH1", None, "rest (weight grads, other tiles)", "AdamW"]
tot = (s[1:, 0] - s[:-1, 0]).mean()
print(f"{tot:.0f} clk/round (CTA {os.environ.get('PRL_TC_PROF_CTA', '0')} with {R} learners resident)")
for i, n in enumerate(names):
    if n is not None:
        j = 8 if i == 7 else i + 1      # stamp 7 is not written: "rest" runs from stamp 6 to stamp 8
        k = 6 if i == 7 else i
        print(f"  {n:36s} {(s[:, j]-s[:, k]).mean():10.0f} clk")
