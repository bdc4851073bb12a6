"""CPU-side checks: the C-ABI library loads and exports every symbol the header
declares (no compute without a GPU), the product fails loudly without CUDA, host
logic (layout arithmetic, error mapping)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "pearl_b200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(prl_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from pearl_b200 import _lib, build
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/pearl_b200.h but not exported"
    # and the ctypes table binds exactly the declared set
    assert sorted(_lib.EXPORTS) == names
    assert _lib.load().prl_abi_version() == 1


def test_layout_arithmetic_is_host_only():
    from pearl_b200 import _lib
    lib = _lib.load()
    d = _lib.BufDesc(1_000_000, 128, 1, 16, _lib.PRL_BUF_DISCRETE)
    lay = _lib.BufLayout()
    assert lib.prl_buf_layout_of(ctypes.byref(d), ctypes.byref(lay)) == 0
    assert lay.record_words * 4 == 1040 and lay.storage_bytes == 1_040_000_000
    assert (lay.off_state, lay.off_next_state, lay.off_action, lay.off_reward, lay.off_flags) == (0, 128, 256, 257, 258)
    d = _lib.BufDesc(10, 6, 1, 5, _lib.PRL_BUF_DISCRETE | _lib.PRL_BUF_DYNAMIC_ACTIONS)
    assert lib.prl_buf_layout_of(ctypes.byref(d), ctypes.byref(lay)) == 0
    assert lay.off_next_state == 8 and lay.record_words % 4 == 0 and lay.off_avail == 19
    d = _lib.BufDesc(10, 376, 17, 0, _lib.PRL_BUF_CONTINUOUS)
    assert lib.prl_buf_layout_of(ctypes.byref(d), ctypes.byref(lay)) == 0
    assert lay.act_words == 17 and lay.record_words * 4 >= 3082
    bad = _lib.BufDesc(0, 4, 1, 2, _lib.PRL_BUF_DISCRETE)
    assert lib.prl_buf_layout_of(ctypes.byref(bad), ctypes.byref(lay)) == _lib.PRL_EINVAL
    with pytest.raises(ValueError):
        _lib.check(lib.prl_buf_layout_of(ctypes.byref(bad), ctypes.byref(lay)))
    assert "capacity" in _lib.last_error()


def test_param_count_matches_torch_module():
    from pearl_b200 import _lib
    lib = _lib.load()
    cfg = _lib.DqnCfg(obs_dim=128, n_actions=16, hidden1=64, hidden2=64, target_update_freq=10, max_batch=256,
                      max_rounds=16)
    assert lib.prl_dqn_param_count(ctypes.byref(cfg)) == 13505
    assert lib.prl_dqn_workspace_bytes(ctypes.byref(cfg)) > 0


def test_slot_expanded_learners_refuse_shapes_past_32_bit_offsets():
    """The conservative and dueling learners index their B (A + 1) slot rows with 32-bit element offsets: a shape with
    max_batch (n_actions + 1) max(slot-expanded width) >= 2^31 is refused by param_count / workspace_bytes (and so by
    create) with a message naming the limit; one row less is accepted.  Host arithmetic only, nothing is allocated."""
    from pearl_b200 import _lib
    lib = _lib.load()
    # 8192 * 256 * 1024 = 2^31: batch 8192, 255 actions, width 1024 (about 32 GB of workspace)
    for B, ok in ((8191, True), (8192, False)):
        cql = _lib.CqlCfg(obs_dim=4, n_actions=255, hidden1=1024, hidden2=7, target_update_freq=10, max_batch=B, max_rounds=1)
        duel = _lib.DuelCfg(obs_dim=4, n_actions=255, feature_dim=3, state_h1=5, state_h2=5, value_h1=5, value_h2=5,
                            adv_h1=7, adv_h2=1024, target_update_freq=10, max_batch=B, max_rounds=1)
        for fn, cfg in ((lib.prl_cql_param_count, cql), (lib.prl_cql_workspace_bytes, cql),
                        (lib.prl_duel_param_count, duel), (lib.prl_duel_workspace_bytes, duel)):
            got = fn(ctypes.byref(cfg))
            if ok:
                assert got > 0, _lib.last_error()
            else:
                assert got == -1 and "2^31" in _lib.last_error()
    ws = lib.prl_cql_workspace_bytes(ctypes.byref(_lib.CqlCfg(obs_dim=4, n_actions=255, hidden1=1024, hidden2=7,
                                                              target_update_freq=10, max_batch=8191, max_rounds=1)))
    assert ws > 2 * 8191 * 256 * 1024 * 4      # c1 and dc1 alone


@pytest.mark.parametrize("max_rounds", [800_000_000, 1 << 30])
def test_workspace_holds_the_per_round_blocks_of_large_max_rounds(max_rounds):
    """max_rounds is only required to be positive: for a max_rounds whose per-round byte counts pass 2^31, every
    learner's workspace still holds its per-round blocks (sampled slots and logical indices, 4 bytes each per row, and the
    float2 AdamW scalars of each optimizer plus, in the DQN family, the int32 target flags).  Host arithmetic only."""
    from pearl_b200 import _lib
    lib = _lib.load()
    small = dict(max_batch=1, max_rounds=max_rounds)
    ac = dict(actor_h1=3, actor_h2=3, critic_h1=3, critic_h2=3)
    cases = [("sac", _lib.SacCfg(obs_dim=2, act_dim=1, **ac, **small), 8 + 2 * 8),
             ("sacd", _lib.SacdCfg(obs_dim=2, n_actions=2, **ac, **small), 8 + 3 * 8),
             ("td3", _lib.Td3Cfg(obs_dim=2, act_dim=1, **ac, actor_update_freq=2, **small), 8 + 2 * 8),
             ("iql", _lib.IqlCfg(obs_dim=2, n_actions=2, **ac, value_h1=3, value_h2=3, **small), 8 + 3 * 8),
             ("ppo", _lib.PpoCfg(obs_dim=2, n_actions=2, **ac, max_rollout=16, **small), 8 + 2 * 8),
             ("qrdqn", _lib.QrdqnCfg(obs_dim=2, n_actions=2, hidden1=3, hidden2=3, num_quantiles=2, target_update_freq=1, **small),
              8 + 8 + 4),
             ("cql", _lib.CqlCfg(obs_dim=2, n_actions=2, hidden1=3, hidden2=3, target_update_freq=1, **small), 8 + 8 + 4),
             ("duel", _lib.DuelCfg(obs_dim=2, n_actions=2, feature_dim=3, state_h1=3, state_h2=3, value_h1=3, value_h2=3, adv_h1=3,
                                   adv_h2=3, target_update_freq=1, **small), 8 + 8 + 4)]
    for name, cfg, bytes_per_round in cases:
        ws = getattr(lib, f"prl_{name}_workspace_bytes")(ctypes.byref(cfg))
        assert ws >= bytes_per_round * max_rounds, (name, ws, _lib.last_error())


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import pearl_b200
    with pytest.raises(RuntimeError):
        pearl_b200.B200ReplayBuffer(16)
    from pearl_b200 import _lib
    assert _lib.load().prl_init(0) != 0  # no device -> error code, never a silent CPU path


def test_product_never_imports_the_oracle():
    """The oracle is a checker: nothing under pearl_b200/ may import, include, load or execute it
    (comments may cite it as the specification)."""
    bad = re.compile(r"^\s*(from|import)\s+oracle\b|#\s*include\s*[\"<][^\">]*oracle|liboracle|CDLL\([^)]*oracle|"
                     r"(subprocess|os\.system|exec|__import__)[^\n]*oracle", re.M)
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pearl_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not bad.search(src), f"{f} uses the oracle"


def test_ctypes_signatures_match_the_header_arity():
    """Every ctypes binding takes exactly as many arguments as the C declaration (a mismatch would corrupt the call
    silently); pointer / integer / floating classes are compared as well."""
    from pearl_b200 import _lib
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"typedef struct[^;{]*\{.*?\}[^;]*;", "", src, flags=re.S)
    decls = dict(re.findall(r"\b(prl_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S))
    assert set(decls) == set(_lib.EXPORTS)

    def kind(c_param: str) -> str:
        p = " ".join(c_param.split())
        if "*" in p or "[" in p:          # arrays decay to pointers
            return "ptr"
        base = p.rsplit(" ", 1)[0] if " " in p else p
        return "float" if base in ("float", "double") else "int"

    def ckind(t) -> str:
        if t in (ctypes.c_float, ctypes.c_double):
            return "float"
        if t in (ctypes.c_int, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint):
            return "int"
        return "ptr"
    for name, params in decls.items():
        plist = [] if params.strip() in ("", "void") else [p for p in params.split(",")]
        _, argtypes = _lib._SIGNATURES[name]
        assert len(plist) == len(argtypes), f"{name}: header has {len(plist)} parameters, ctypes table {len(argtypes)}"
        for i, (cp, at) in enumerate(zip(plist, argtypes)):
            assert kind(cp) == ckind(at), f"{name} argument {i}: `{' '.join(cp.split())}` bound as {at}"
