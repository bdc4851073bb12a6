"""The image-observation path of B200DeepQLearning / B200DoubleDQN: Pearl's DeepQLearning / DoubleDQN built with a
`network_instance` of CNNQValueNetwork or CNNQValueMultiHeadNetwork (the Atari DQN configurations), on an H100 through
`prl_cnnq_*` (csrc/cnnq.cu).

The DQN plugin (dqn.py) keeps its binding: `_Q`, `_Q_target` and the AdamW state are views into the flat vectors it
allocates, and a checkpoint or lr change is picked up the same way.  A state is a [C, H, W] tensor of pixel values; the
replay ring stores it flattened in (c, h, w) order, as B200ReplayBuffer stores any state, and the trunk divides it by 255
as the reference does.  As in the reference, `learn_batch` and `act` take 4-D states only ([B, C, H, W] and
[1, C, H, W]).  The multi-head network reproduces the reference's [B, B] broadcast of its MSE loss (include/pearl_b200.h).
No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._batch import dense_rows, next_available_first, plugin_call
from ._compat import CNNQValueMultiHeadNetwork, CNNQValueNetwork
from .replay_buffer import _stream_ptr

PREFIX = "prl_cnnq_"
NAME = "CNN DQN"
LAUNCH_INFO = dict(launches="last_launches")
MAX_CONV, MAX_FC, MAX_ACTIONS = 4, 2, 255


def is_cnn(qnet) -> bool:
    """By class: both of Pearl's CNN Q networks."""
    return isinstance(qnet, (CNNQValueNetwork, CNNQValueMultiHeadNetwork))


def _square(v, what: str) -> int:
    t = tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    if len(t) != 2 or t[0] != t[1]:
        raise NotImplementedError(f"pearl_b200 fuses square conv {what}s only; got {t}")
    return int(t[0])


def shape_of(qnet, n_actions: int) -> dict:
    """The trunk and FC shape of a CNN Q network: input (C, H, W), conv layers (out-channels, kernel, stride, padding),
    the hidden FC widths and whether it is the multi-head network.  `_model_cnn` must be Conv2d+ReLU layers (1 to 4),
    `_model_fc` Linear+ReLU blocks (0 to 2) and a Linear with 1 (vanilla) or n_actions (multi-head) outputs."""
    multi = isinstance(qnet, CNNQValueMultiHeadNetwork)
    cnn, fc = getattr(qnet, "_model_cnn", None), getattr(qnet, "_model_fc", None)
    if not isinstance(cnn, torch.nn.Module) or not isinstance(fc, torch.nn.Module):
        raise NotImplementedError("pearl_b200 fuses CNN Q networks whose layers are their `_model_cnn` / `_model_fc` blocks")
    leaves = lambda m: [x for x in m.modules() if not isinstance(x, torch.nn.Sequential)]  # noqa: E731
    cmods, fmods = leaves(cnn), leaves(fc)
    if any(isinstance(m, (torch.nn.BatchNorm2d, torch.nn.BatchNorm1d)) for m in cmods + fmods):
        raise NotImplementedError("batch norm: pearl_b200 fuses CNN Q networks without batch norm")
    ckinds = [type(m) for m in cmods]
    if len(cmods) % 2 or ckinds != [torch.nn.Conv2d, torch.nn.ReLU] * (len(cmods) // 2):
        raise NotImplementedError(f"pearl_b200 fuses conv trunks of Conv2d+ReLU layers; got {[k.__name__ for k in ckinds]}")
    convs = cmods[0::2]
    if not 1 <= len(convs) <= MAX_CONV:
        raise NotImplementedError(f"pearl_b200 fuses 1 to {MAX_CONV} conv layers; got {len(convs)}")
    fkinds = [type(m) for m in fmods]
    n_hidden = (len(fmods) - 1) // 2
    if len(fmods) % 2 == 0 or fkinds != [torch.nn.Linear, torch.nn.ReLU] * n_hidden + [torch.nn.Linear]:
        raise NotImplementedError("pearl_b200 fuses FC stacks of Linear+ReLU layers and a Linear head; got "
                                  f"{[k.__name__ for k in fkinds]}")
    if n_hidden > MAX_FC:
        raise NotImplementedError(f"pearl_b200 fuses at most {MAX_FC} hidden fully connected layers; got {n_hidden}")
    C, H, W = int(qnet._input_channels), int(qnet._input_height), int(qnet._input_width)
    layers, c, h, w = [], C, H, W
    for m in convs:
        if m.groups != 1 or _square(m.dilation, "dilation") != 1 or m.padding_mode != "zeros" or m.bias is None:
            raise NotImplementedError("pearl_b200 fuses plain Conv2d layers (groups 1, dilation 1, zero padding, bias)")
        k, s, p = _square(m.kernel_size, "kernel"), _square(m.stride, "stride"), _square(m.padding, "padding")
        if m.in_channels != c:
            raise NotImplementedError("unexpected conv trunk: a layer's in-channels differ from the previous out-channels")
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        if h < 1 or w < 1:
            raise ValueError("a conv layer's output would be empty: every conv output must be at least 1 x 1")
        layers.append((int(m.out_channels), k, s, p))
        c = m.out_channels
    lins = fmods[0::2]
    F = c * h * w
    if lins[0].in_features != F + (0 if multi else n_actions):
        raise NotImplementedError("unexpected CNN Q-network shape: the FC input must be the conv features"
                                  + ("" if multi else " and the one-hot action"))
    out = n_actions if multi else 1
    if lins[-1].out_features != out:
        raise NotImplementedError(f"unexpected CNN Q-network shape: the head must have {out} output(s)")
    return dict(input=(C, H, W), conv=layers, hidden=[int(m.out_features) for m in lins[:-1]], multi=multi)


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the CNN configurations the CUDA learner does not run."""
    if pl._sarsa:
        raise NotImplementedError("DeepSARSA with a CNN Q network is not supported")
    if pl._conservative:
        raise NotImplementedError("conservative (CQL) updates with a CNN Q network are not supported")
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no CNN kernel: use engine='auto' or 'simt'")
    if pl._n_actions > MAX_ACTIONS:
        raise ValueError(f"a CNN Q network needs at most {MAX_ACTIONS} actions: next-action ids are stored as bytes")
    pl._adam_hparams()


def learn_args(pl) -> tuple:
    """prl_cnnq_learn takes nothing after the training-step count."""
    return ()


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.CnnqCfg:
    sh = pl._cnn
    conv = sh["conv"] + [(0, 0, 0, 0)] * (MAX_CONV - len(sh["conv"]))
    arr = lambda i: (C.c_int32 * MAX_CONV)(*[c[i] for c in conv])  # noqa: E731
    hidden = sh["hidden"] + [0] * (MAX_FC - len(sh["hidden"]))
    return _lib.CnnqCfg(in_c=sh["input"][0], in_h=sh["input"][1], in_w=sh["input"][2], n_conv=len(sh["conv"]),
                        conv_out=arr(0), conv_kernel=arr(1), conv_stride=arr(2), conv_pad=arr(3), n_fc=len(sh["hidden"]),
                        fc_hidden=(C.c_int32 * MAX_FC)(*hidden), n_actions=pl._n_actions, multi_head=int(sh["multi"]),
                        double_dqn=int(pl._double), target_update_freq=int(pl._target_update_freq), max_batch=max_batch,
                        max_rounds=pl._max_rounds, lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"],
                        weight_decay=hp["weight_decay"], gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def _images(pl, t: torch.Tensor, what: str, lead=None) -> torch.Tensor:
    """`t` as [N, C, H, W]: the reference's get_q_values asserts a 4-D state batch."""
    shape = tuple(pl._cnn["input"])
    if t.dim() != 4 or tuple(t.shape[1:]) != shape or (lead is not None and t.shape[0] != lead):
        n = "N" if lead is None else lead
        raise ValueError(f"{what} must be [{n}, {', '.join(map(str, shape))}] (the reference's CNN Q networks take 4-D states); "
                         f"got {list(t.shape)}")
    return t


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` on a caller-supplied batch: state / next_state [B, C, H, W], actions as raw ids or
    one-hot rows.  Next-action slots that are masked are compacted away in order, which keeps DoubleDQN's first argmax."""
    B, A = len(batch), pl._n_actions
    _images(pl, torch.as_tensor(batch.state), "batch.state", B)
    _images(pl, torch.as_tensor(batch.next_state), "batch.next_state", B)
    pl._bind(B)
    dev = pl._device
    return plugin_call(pl, B, *dense_rows(batch, B, A, dev), *next_available_first(batch, B, A, dev), int(pl._training_steps))


def q_values(pl, states: torch.Tensor, target: bool = False) -> torch.Tensor:
    """Q(s, a) for every action id: [N, C, H, W] -> [N, n_actions]."""
    s = _images(pl, torch.as_tensor(states), "states")
    pl._bind(1)
    dev = pl._device
    s = s.to(device=dev, dtype=torch.float32).contiguous()
    out = torch.empty((s.shape[0], pl._n_actions), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(pl._c("q_values")(pl._handle, s.shape[0], _lib.ptr(s), int(target), _lib.ptr(out), _stream_ptr(dev)))
    torch.cuda.current_stream(dev).synchronize()
    return out


def act_values(pl, subjective_state) -> torch.Tensor:
    """The Q values DeepTDLearning.act computes: for a [1, C, H, W] state, [n_actions].  A [C, H, W] state is refused
    before any device call, as the reference's get_q_values asserts a 4-D state (act adds a batch axis to 1-D states only)."""
    s = torch.as_tensor(subjective_state)
    _images(pl, s, "the state act() takes", 1)
    return q_values(pl, s)[0]
