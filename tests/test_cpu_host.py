"""CPU-only tests (`pytest -m "not gpu"`): the C restatement of the oracle against the torch port,
the C-ABI library (loads, exports every symbol include/aa_b200.h declares), the host-side row
planning, the packed all-reduce over gloo with world_size 2, and the no-CPU-fallback contract."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import c_oracle
from oracle import ref_port as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(a, t):
    return a.ctypes.data_as(ctypes.POINTER(t))


def test_c_oracle_token_log_probs_and_grad():
    lib = c_oracle.lib()
    gen = torch.Generator().manual_seed(0)
    rows, V = 7, 1031
    x = (torch.randn(rows, V, generator=gen) * 2.5)
    y = torch.randint(0, V, (rows,), generator=gen)
    out = np.zeros(rows)
    xa, ya = x.numpy().copy(), y.numpy().copy()
    lib.oracle_token_log_probs(_p(xa, ctypes.c_float), _p(ya, ctypes.c_int64), ctypes.c_int64(rows),
                               ctypes.c_int64(V), _p(out, ctypes.c_double))
    want = O.token_log_probs(x.double().unsqueeze(0), y.unsqueeze(0))[0]
    assert np.allclose(out, want.numpy(), rtol=0, atol=1e-12)
    g = torch.randn(rows, generator=gen).double()
    grad = np.zeros((rows, V))
    ga = g.numpy().copy()
    lib.oracle_token_log_probs_grad(_p(xa, ctypes.c_float), _p(ya, ctypes.c_int64), _p(ga, ctypes.c_double),
                                    ctypes.c_int64(rows), ctypes.c_int64(V), _p(grad, ctypes.c_double))
    leaf = x.double().requires_grad_(True)
    O.token_log_probs(leaf.unsqueeze(0), y.unsqueeze(0))[0].backward(g)
    assert np.allclose(grad, leaf.grad.numpy(), atol=1e-12)


def test_c_oracle_dpo_pair_vs_port():
    lib = c_oracle.lib()
    lib.oracle_dpo_pair.argtypes = [ctypes.c_double] * 5 + [ctypes.POINTER(ctypes.c_double)] * 3
    gen = torch.Generator().manual_seed(1)
    lp = -torch.rand(4, 9, generator=gen).double() * 5
    rlp = lp + 0.3 * torch.randn(4, 9, generator=gen).double()
    want = O.dpo_loss(lp, rlp, 0.1)
    for i in range(2):
        a, b, c = ctypes.c_double(), ctypes.c_double(), ctypes.c_double()
        lib.oracle_dpo_pair(float(lp[i].sum()), float(lp[2 + i].sum()), float(rlp[i].sum()), float(rlp[2 + i].sum()),
                            0.1, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        assert abs(b.value - float(want['better_sample_reward'][i])) < 1e-12
        assert abs(c.value - float(want['worse_sample_reward'][i])) < 1e-12
    # mean of the two pair losses
    tot = 0.0
    for i in range(2):
        a, b, c = ctypes.c_double(), ctypes.c_double(), ctypes.c_double()
        lib.oracle_dpo_pair(float(lp[i].sum()), float(lp[2 + i].sum()), float(rlp[i].sum()), float(rlp[2 + i].sum()),
                            0.1, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        tot += a.value
    assert abs(tot / 2 - float(want['loss'])) < 1e-12


def test_c_oracle_ppo_and_layout(golden):
    lib = c_oracle.lib()
    c = golden('ppo')['f32']
    hp = O.PPO_DEFAULTS
    B, W = c['log_probs'].shape
    for b in range(B):
        lp, ref = c['log_probs'][b].double().numpy().copy(), c['ref_log_probs'][b].double().numpy().copy()
        mask = c['mask'][b].to(torch.uint8).numpy().copy()
        out = np.zeros(W)
        end = lib.oracle_kl_rewards(_p(lp, ctypes.c_double), _p(ref, ctypes.c_double), _p(mask, ctypes.c_uint8),
                                    ctypes.c_int64(W), ctypes.c_double(float(c['reward'][b])),
                                    ctypes.c_double(hp['kl_coeff']), ctypes.c_double(hp['clip_range_score']),
                                    _p(out, ctypes.c_double))
        assert end == int(c['mask'][b].nonzero()[-1])
        assert np.allclose(out, c['rewards'][b].double().numpy(), atol=1e-6)
        s = c['start']
        adv, ret = np.zeros(W - s), np.zeros(W - s)
        vals = c['values'][b].double().numpy().copy()
        rew = c['rewards'][b].double().numpy().copy()
        lib.oracle_gae(_p(vals, ctypes.c_double), _p(rew, ctypes.c_double), _p(mask, ctypes.c_uint8), ctypes.c_int64(W),
                       ctypes.c_int64(s), ctypes.c_double(hp['gamma']), ctypes.c_double(hp['gae_lambda']),
                       _p(adv, ctypes.c_double), _p(ret, ctypes.c_double))
        assert np.allclose(adv, c['advantages'][b].double().numpy(), atol=1e-5)
        assert np.allclose(ret, c['returns'][b].double().numpy(), atol=1e-5)
    g = golden('layout')
    ids = g['ids'].numpy().copy()
    out = np.zeros_like(ids)
    lib.oracle_move_padding_left(_p(ids, ctypes.c_int64), ctypes.c_int64(ids.shape[0]), ctypes.c_int64(ids.shape[1]),
                                 ctypes.c_int64(g['pad']), _p(out, ctypes.c_int64))
    assert np.array_equal(out, g['moved'].numpy())
    for i, want in enumerate(g['stripped']):
        R = len(want)
        if R == 0:
            continue
        buf = np.zeros(R, dtype=np.int64)
        row = ids[i].copy()
        n = lib.oracle_strip_pad_tail(_p(row, ctypes.c_int64), ctypes.c_int64(len(row)), ctypes.c_int64(g['pad']),
                                      ctypes.c_int64(R), _p(buf, ctypes.c_int64))
        assert n == R and np.array_equal(buf, want.numpy())


# ---- the C-ABI library ---------------------------------------------------------------------------
def test_library_exports_every_declared_symbol():
    from align_anything_b200 import _lib, build

    path = build.build()
    header = open(os.path.join(ROOT, 'include', 'aa_b200.h')).read()
    declared = set(re.findall(r'^(?:int|const char \*)\s*\*?(aa_\w+)\s*\(', header, flags=re.M))
    assert len(declared) >= 18, declared
    handle = ctypes.CDLL(path)
    missing = [s for s in declared if not hasattr(handle, s)]
    assert not missing, missing
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    m = re.search(r"#define AA_B200_ABI_VERSION (\d+)", header)
    assert handle.aa_abi_version() == int(m.group(1)) == 3
    # only sm_90a code in the binary
    r = subprocess.run(['cuobjdump', '-lelf', path], capture_output=True, text=True)
    if r.returncode == 0 and r.stdout.strip():
        assert 'sm_90a' in r.stdout and not re.search(r'sm_(?!90a)\d+', r.stdout), r.stdout


def test_argument_errors_need_no_gpu():
    from align_anything_b200 import _lib

    lib = _lib.lib()
    rc = lib.aa_logprob_fwd(None, 0, 0, 0, None, 0, 0, 1, 1, None, None, None, None, None, 0, None, None, None, None)
    assert rc == -2 and b'bad sizes' in lib.aa_last_error()
    rc = lib.aa_logprob_set_tuning(7, 0)  # kernel digit 7 is invalid
    assert rc == -2
    assert lib.aa_logprob_set_tuning(12, 0) == -2  # a variant names a kernel (0..3); there are no shape codes
    assert lib.aa_logprob_set_tuning_bwd(2, 0) == -2  # backward kernels: -1 / 0 / 1 (TMA-staged), 3 (LDG)
    assert lib.aa_logprob_set_tuning_bwd(11, 0) == -2
    with pytest.raises(RuntimeError):
        _lib.check(rc)
    # entry points added later in the round: argument validation happens before any CUDA call
    buf = (ctypes.c_int64 * 4)(0, 1, 2, 3)
    ptr = ctypes.cast(buf, ctypes.c_void_p)
    assert lib.aa_linear_logprob_fwd(None, 0, 64, 64, None, 10, 64, None, None, 0, None, None, None, 0, 0, None, None) == 0  # 0 rows
    rc = lib.aa_linear_logprob_fwd(ptr, 4, 100, 104, ptr, 10, 104, ptr, ptr, 0, None, None, None, 0, 0, None, None)
    assert rc == -4 and b"multiple of 64" in lib.aa_last_error()  # AA_ERR_UNSUPPORTED
    rc = lib.aa_linear_logprob_fwd(None, 4, 64, 64, ptr, 10, 64, ptr, ptr, 0, None, None, None, 0, 0, None, None)
    assert rc == -2 and b'null pointer' in lib.aa_last_error()
    rc = lib.aa_linear_logprob_fwd(ptr, 4, 64, 60, ptr, 10, 64, ptr, ptr, 0, None, None, None, 0, 0, None, None)
    assert rc == -3 and b"16-byte" in lib.aa_last_error()  # AA_ERR_ALIGN: row stride 60 elements
    assert lib.aa_zero_rows(None, 0, 8, 8, 4, None, 0, None) == 0  # no spans
    rc = lib.aa_zero_rows(ptr, 0, 4, 8, 4, ptr, 1, None)
    assert rc == -2 and b'bad sizes' in lib.aa_last_error()  # row_stride < V
    rc = lib.aa_tail_rows(ptr, 0, 8, ptr, 2, 8, 9, ptr, 9, 0, None)
    assert rc == -2 and b'Rmax=9' in lib.aa_last_error()  # Rmax > W
    rc = lib.aa_logprob_bwd(ptr, 0, 8, 8, ptr, 0, 0, 1, 1, ptr, ptr, ptr, ptr, ptr, ptr, ptr, None, 0, None, None, 2, ptr, 8, 4,
                            ptr, 2, None, 0, None)
    assert rc == -2 and b'extra_zero_rows' in lib.aa_last_error()  # listed rows only with n_tile_rows == 0


def test_no_cpu_fallback():
    from align_anything_b200 import ops
    from align_anything_b200.utils import tools

    with pytest.raises(RuntimeError, match='no CPU fallback'):
        tools.gather_log_probabilities(torch.randn(1, 3, 8), torch.zeros(1, 3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        ops.move_padding_left(torch.zeros(2, 4, dtype=torch.int64), 0)
    # nothing under the package imports the oracle
    pkg = os.path.join(ROOT, 'align_anything_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r'^\s*(from|import)\s+oracle', src, flags=re.M), f


# ---- host-side planning ----------------------------------------------------------------------------
def test_row_plans():
    from align_anything_b200 import ops

    # DPO tails: sample i scores R_i - 1 rows starting at L - R_i, labels from column 1 of its label row
    plan = ops._tail_plan((5, 2, 7), 16, 16 * 100, 100, 7, 1, 0, None, 'cpu')
    t = plan.dev
    assert plan.n_rows == 4 + 1 + 6 and plan.out_shape == (3, 6) and plan.n_tile_rows == 48
    assert t[0, :3].tolist() == [11 * 100, 1600 + 14 * 100, 3200 + 9 * 100]
    assert t[1, :3].tolist() == [1, 8, 15]
    assert t[2, :3].tolist() == [0, 6, 12]
    assert t[3].tolist() == [0, 4, 5, 11]
    assert t[4, :3].tolist() == [11, 30, 41]
    # multimodal PPO tails: R rows starting at L - R - 1
    plan = ops._tail_plan((5, 2), 16, 1600, 100, 5, 0, -1, None, 'cpu')
    assert plan.dev[3].tolist() == [0, 5, 7] and plan.dev[4, :2].tolist() == [10, 29]
    # dense view logits[:, :-1] of a contiguous (2, 8, V) base: two segments, tile rows in the base
    plan = ops._dense_plan(2, 7, 8 * 50, 50, 8, 0, 8, 16, 'cpu')
    assert plan.n_seg == 2 and plan.dev[4, :2].tolist() == [0, 8] and plan.dev[0, :2].tolist() == [0, 400]
    # fully contiguous: collapses to one segment
    plan = ops._dense_plan(2, 8, 400, 50, 8, 0, 8, 16, 'cpu')
    assert plan.n_seg == 1 and plan.n_rows == 16


def test_reroute_detection():
    from align_anything_b200 import ops

    base = torch.randn(3, 9, 13)
    assert ops._try_reroute(base[:, :-1])[1] == 0
    assert ops._try_reroute(base[1][-4:].unsqueeze(0)[:, :-1]) == (base, 9 + 5) or True
    r = ops._try_reroute(base[1][-4:].unsqueeze(0)[:, :-1])
    assert r is not None and r[0] is base and r[1] == 14
    assert ops._try_reroute(base) is None  # not a view
    assert ops._try_reroute(base[:, :, :5]) is None  # vocab slice: rows not whole


_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["AA_ROOT"])
from align_anything_b200.utils.multi_process import all_reduce_packed, get_all_reduce_mean, get_all_reduce_max
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + os.environ["AA_PORT"],
                        rank=int(os.environ["RANK"]), world_size=2)
r = dist.get_rank()
stats = torch.tensor([1.0 + r, 10.0 * (r + 1), 3.0, float(5 + 4 * r)])
out = all_reduce_packed(stats.clone(), max_lanes=(3,))
assert out.tolist() == [1.5, 15.0, 3.0, 9.0], out
out = all_reduce_packed(stats.clone())
assert out.tolist() == [1.5, 15.0, 3.0, 7.0], out
assert float(get_all_reduce_mean(torch.tensor(float(r)))) == 0.5
assert float(get_all_reduce_max(torch.tensor(float(r)))) == 1.0
# Safe RLHF-V lambda step across ranks (saferlhf.py:487-500): episode cost averaged onto rank 0, SGD there, broadcast
import math
from collections import deque
from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer
tr = SafeRLHFVTrainer(None)
tr.log_lambda = torch.nn.Parameter(torch.tensor(math.log(2.0)))
tr.log_lambda_optimizer = torch.optim.SGD([tr.log_lambda], lr=0.1)
tr.log_lambda_max, tr.threshold, tr.lambda_update_delay_steps, tr.global_step = None, 0.5, 0, 1
tr.episode_costs = deque([1.0 + 2.0 * r], maxlen=4)   # rank means 1 and 3 -> global mean 2
tr._lambda_step()
want = math.log(2.0) + 0.1 * (2.0 - 0.5) * 2.0
assert abs(tr.log_lambda.item() - want) < 1e-6, (r, tr.log_lambda.item(), want)
dist.destroy_process_group()
print("ok", r)
'''


def test_packed_all_reduce_gloo_world2(tmp_path):
    """N > 1 host logic on CPU: one collective carries AVG lanes and a MAX lane."""
    import socket

    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    script = tmp_path / 'worker.py'
    script.write_text(_WORKER)
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), AA_PORT=str(port), AA_ROOT=ROOT)
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    for p in procs:
        out, _ = p.communicate(timeout=180)
        assert p.returncode == 0, out


def test_saferlhf_lambda_step_matches_reference_update():
    """saferlhf.py:487-500: one SGD step on log_lambda with loss -(J_C - d) * exp(log_lambda), clamp at log_lambda_max."""
    import math
    from collections import deque

    from align_anything_b200.trainers.text_image_to_text.saferlhf import SafeRLHFVTrainer

    tr = SafeRLHFVTrainer(None)
    tr.log_lambda = torch.nn.Parameter(torch.tensor(math.log(2.0)))
    tr.log_lambda_optimizer = torch.optim.SGD([tr.log_lambda], lr=0.1)
    tr.log_lambda_max, tr.threshold, tr.lambda_update_delay_steps, tr.global_step = math.log(5.0), 0.5, 0, 3
    tr.episode_costs = deque([1.0, 2.0, 3.0], maxlen=8)
    tr._lambda_step()
    want = math.log(2.0) + 0.1 * (2.0 - 0.5) * 2.0
    assert abs(tr.log_lambda.item() - want) < 1e-6
    tr.episode_costs.extend([100.0] * 8)
    tr._lambda_step()
    assert abs(tr.log_lambda.item() - math.log(5.0)) < 1e-6  # clamped
    tr.global_step, tr.lambda_update_delay_steps = 0, 10
    before = tr.log_lambda.item()
    tr._lambda_step()
    assert tr.log_lambda.item() == before  # delayed


def test_row_plan_zero_spans_are_the_complement_of_the_segments():
    from align_anything_b200.ops import RowPlan

    # three segments inside a 100-row tile: rows [20, 30), [31, 50), [90, 100)
    plan = RowPlan([0, 0, 0], [0, 0, 0], [0, 0, 0], [10, 19, 10], [20, 31, 90], (3, 19), 100, torch.device('cpu'))
    spans = [(plan.zero_spans[2 * i], plan.zero_spans[2 * i + 1]) for i in range(plan.n_zero_spans)]
    assert spans == [(0, 20), (50, 40)]          # long spans: copy engine
    assert plan.extra_zero_rows.tolist() == [30]  # isolated row: listed for the kernel
    assert plan.n_extra == 1 and plan.n_rows == 39
    covered = sum(n for _, n in spans) + plan.n_extra + plan.n_rows
    assert covered == 100
    with pytest.raises(ValueError, match='overlap'):
        RowPlan([0, 0], [0, 0], [0, 0], [10, 10], [0, 5], (2, 10), 40, torch.device('cpu'))
    dense = RowPlan([0], [0], [0], [64], [0], (64,), 0, torch.device('cpu'))
    assert dense.n_zero_spans == 0 and dense.n_extra == 0


def test_row_plan_zero_spans_partition_property():
    """Random segment layouts: scored rows + memset spans + listed rows partition the gradient tile exactly once."""
    from hypothesis import given, settings
    from hypothesis import strategies as st

    from align_anything_b200.ops import RowPlan

    @settings(max_examples=60, deadline=None)
    @given(st.lists(st.tuples(st.integers(0, 40), st.integers(0, 50)), min_size=1, max_size=12), st.integers(0, 40))
    def check(gaps_and_counts, tail_gap):
        tile_row, counts, at = [], [], 0
        for gap, n in gaps_and_counts:
            at += gap
            tile_row.append(at)
            counts.append(n)
            at += n
        n_tile = at + tail_gap
        if n_tile == 0:
            return
        k = len(counts)
        plan = RowPlan([0] * k, [0] * k, [0] * k, counts, tile_row, (k, max(counts + [1])), n_tile, torch.device('cpu'))
        seen = [0] * n_tile
        for first, n in zip(tile_row, counts):
            for r in range(first, first + n):
                seen[r] += 1
        for i in range(plan.n_zero_spans):
            first, n = plan.zero_spans[2 * i], plan.zero_spans[2 * i + 1]
            assert n >= RowPlan.MEMSET_MIN_ROWS
            for r in range(first, first + n):
                seen[r] += 1
        if plan.n_extra:
            for r in plan.extra_zero_rows.tolist():
                seen[r] += 1
        assert all(c == 1 for c in seen), seen
        assert plan.n_rows == sum(counts)

    check()


def test_c_oracle_sibling_losses_vs_port():
    """The independent fp64 C restatement of SimPO / ORPO / KTO / RM / GRPO / Safe RLHF-V against the torch port
    (which is pinned bit-exactly on goldens of the unmodified reference) evaluated in float64."""
    lib = c_oracle.lib()
    D, PD = ctypes.c_double, ctypes.POINTER(ctypes.c_double)
    gen = torch.Generator().manual_seed(4)
    B, L_, pad = 3, 14, 0
    ids = torch.randint(2, 50, (2 * B, L_), generator=gen)
    for i in range(B):  # shared prefix of 5 tokens, then the pair diverges
        ids[B + i, :5] = ids[i, :5]
    ids[0, 11:] = pad
    ids[B + 2, 9:] = pad
    mask = ids != pad
    lp = -torch.rand(2 * B, L_, generator=gen, dtype=torch.float64) * 0.5 - 0.05
    rlp = lp + 0.1 * torch.randn(2 * B, L_, generator=gen, dtype=torch.float64)
    beta, gamma = 0.1, 0.5
    simpo = O.simpo_loss(lp, ids, mask, beta, gamma)
    orpo = O.orpo_loss(lp, ids, mask, beta)
    kto = O.kto_loss(lp, rlp, ids, mask, beta, 1.0, 1.33, 0.07)
    s_l, o_l, k_l = [], [], []
    for i in range(B):
        div = int((ids[i] != ids[B + i]).nonzero()[0])
        eb, ew = int(mask[i].nonzero()[-1]), int(mask[B + i].nonzero()[-1])
        bs, ws = float(lp[i, div:eb + 1].sum()), float(lp[B + i, div:ew + 1].sum())
        rbs, rws = float(rlp[i, div:eb + 1].sum()), float(rlp[B + i, div:ew + 1].sum())
        out = [D() for _ in range(3)]
        lib.oracle_simpo_pair(D(bs), D(ws), D(eb + 1), D(ew + 1), D(beta), D(gamma), *[ctypes.byref(o) for o in out])
        s_l.append(out[0].value)
        assert abs(out[1].value - float(simpo['better_sample_reward'][i])) < 1e-12
        lib.oracle_orpo_pair(D(bs), D(ws), D(eb + 1), D(ew + 1), D(beta), *[ctypes.byref(o) for o in out])
        o_l.append(out[0].value)
        lib.oracle_kto_pair(D(bs), D(rbs), D(ws), D(rws), D(beta), D(1.0), D(1.33), D(0.07), *[ctypes.byref(o) for o in out])
        k_l.append(out[0].value)
        assert abs(out[2].value - float(kto['worse_sample_reward'][i])) < 1e-12
    assert abs(sum(s_l) / B - float(simpo['loss'])) < 1e-12
    assert abs(sum(o_l) / B - float(orpo['loss'])) < 1e-12
    assert abs(sum(k_l) / B - float(kto['loss'])) < 1e-12
    # RM pairwise loss
    hi, lo = torch.randn(5, generator=gen, dtype=torch.float64), torch.randn(5, generator=gen, dtype=torch.float64)
    want = -torch.nn.functional.logsigmoid(hi - lo)
    for i in range(5):
        assert abs(lib.oracle_rm_pair(D(float(hi[i])), D(float(lo[i]))) - float(want[i])) < 1e-12
    # GRPO: group advantages, per-token loss and its gradient
    rewards = torch.randn(8, generator=gen, dtype=torch.float64)
    adv = np.zeros(8)
    ra = rewards.numpy().copy()
    lib.oracle_group_advantages(ra.ctypes.data_as(PD), ctypes.c_int64(2), ctypes.c_int64(4), adv.ctypes.data_as(PD))
    assert np.allclose(adv, O.grpo_group_advantages(rewards, 2, 4).view(-1).numpy(), atol=1e-12)
    tok_lp = (-torch.rand(1, 6, generator=gen, dtype=torch.float64)).requires_grad_(True)
    tok_ref = tok_lp.detach() + 0.2 * torch.randn(1, 6, generator=gen, dtype=torch.float64)
    seqs = torch.randint(3, 20, (1, 10), generator=gen)  # no eos (id 1): every completion token counts
    loss = O.grpo_loss(tok_lp, tok_ref, torch.tensor([[0.7]], dtype=torch.float64), seqs, 4, 1, 0.04)
    loss.backward()
    tot = 0.0
    for t in range(6):
        out = [D() for _ in range(3)]
        lib.oracle_grpo_token(D(float(tok_lp.detach()[0, t])), D(float(tok_ref[0, t])), D(0.7), D(0.04), *[ctypes.byref(o) for o in out])
        tot += out[1].value
        assert abs(out[2].value / 6 - float(tok_lp.grad[0, t])) < 1e-12
    assert abs(tot / 6 - float(loss.detach())) < 1e-12
    # Safe RLHF-V actor loss
    n = 7
    a = {k: torch.randn(1, n, generator=gen, dtype=torch.float64) for k in ('lp', 'old', 'ra', 'ca')}
    a['lp'] = a['old'] + 0.3 * torch.randn(1, n, generator=gen, dtype=torch.float64)
    want = O.saferlhf_actor_loss(a['lp'], a['old'], a['ra'], a['ca'], torch.ones(1, n, dtype=torch.bool), 1.7, 0.2)
    got = sum(lib.oracle_saferlhf_actor_token(D(float(a['lp'][0, t])), D(float(a['old'][0, t])), D(float(a['ra'][0, t])),
                                              D(float(a['ca'][0, t])), D(1.7), D(0.2)) for t in range(n)) / n
    assert abs(got - float(want)) < 1e-12


def test_hidden_state_row_gather_matches_the_reference_row_selection(monkeypatch):
    """Host logic of the lm_head paths (ops._tails_from_hidden): which hidden rows are scored against which labels.
    The CUDA pieces are replaced by torch stand-ins here (test-only monkeypatching), the index arithmetic is the real one:
    DPO rows (trainers/text_to_text/dpo.py:133-142) and multimodal PPO tails (text_image_to_text/ppo.py:233-246)."""
    from align_anything_b200 import ops

    def fake_linear_lp(hidden, weight, labels, chunk_rows=None, mode=None):
        return O.token_log_probs(torch.nn.functional.linear(hidden, weight).unsqueeze(0), labels.unsqueeze(0))[0]

    def fake_strip(input_ids, lens, pad_id, strip=True):
        out = torch.zeros((input_ids.size(0), max(lens)), dtype=torch.int64)
        for i, r in enumerate(lens):
            row = input_ids[i][input_ids[i] != pad_id] if strip else input_ids[i]
            out[i, :r] = row[-r:]
        return out

    monkeypatch.setattr(ops.L, 'require_cuda', lambda *a: None)
    monkeypatch.setattr(ops, 'linear_token_log_probs', fake_linear_lp)
    monkeypatch.setattr(ops, 'strip_pad_tail', fake_strip)
    monkeypatch.setattr(ops, '_lens_tensor', lambda lens, dev: torch.tensor(lens, dtype=torch.int32))
    gen = torch.Generator().manual_seed(2)
    n, L_, H, V, pad = 4, 18, 8, 37, 36
    lens = [5, 11, 2, 8]
    ids = torch.randint(2, pad, (n, L_), generator=gen)
    for i, r in enumerate(lens):
        ids[i, : L_ - r - 3] = pad
    hidden = torch.randn(n, L_, H, generator=gen)
    weight = torch.randn(V, H, generator=gen)
    logits = torch.nn.functional.linear(hidden, weight)
    got = ops.sequence_log_probs_from_hidden(hidden, weight, ids, lens, pad)
    want = O.dpo_sequence_log_probs(logits, ids, lens, pad, True)
    assert got.shape == want.shape and torch.allclose(got, want, atol=1e-5)
    got_mm = ops.tail_log_probs_from_hidden(hidden, weight, ids, lens)
    rows = [O.token_log_probs(logits[b, :-1][-r:].unsqueeze(0), ids[b, 1:][-r:].unsqueeze(0)).squeeze(0) for b, r in enumerate(lens)]
    want_mm = torch.nn.utils.rnn.pad_sequence(rows, batch_first=True)
    assert got_mm.shape == want_mm.shape and torch.allclose(got_mm, want_mm, atol=1e-5)
    w_pad, Vp = ops._pad_vocab(weight.bfloat16())
    assert Vp == 40 and torch.equal(w_pad[:V], weight.bfloat16()) and float(w_pad[V:].abs().max()) == 0.0


def test_fused_lm_head_refuses_heads_it_would_get_wrong():
    """ADVICE r1: the fused lm_head paths read the head weight outside the module forward and model a plain bias-free
    projection -- ZeRO-3 placeholders, biased heads and soft-capped / scaled logits must fail loudly, not silently."""
    from types import SimpleNamespace

    from align_anything_b200 import ops

    w = torch.zeros(8, 4)
    ok = SimpleNamespace(get_output_embeddings=lambda: SimpleNamespace(weight=w, bias=None), config=SimpleNamespace())
    assert ops.lm_head_weight(ok) is w
    z3 = torch.zeros(0)
    z3.ds_id = 7
    for bad, msg in (
        (SimpleNamespace(get_output_embeddings=lambda: SimpleNamespace(weight=z3, bias=None)), 'ZeRO-3'),
        (SimpleNamespace(get_output_embeddings=lambda: SimpleNamespace(weight=w, bias=torch.zeros(8))), 'bias-free'),
        (SimpleNamespace(get_output_embeddings=lambda: SimpleNamespace(weight=w, bias=None),
                         config=SimpleNamespace(final_logit_softcapping=30.0)), 'final_logit_softcapping'),
        (SimpleNamespace(get_output_embeddings=lambda: SimpleNamespace(weight=w, bias=None),
                         config=SimpleNamespace(logit_scale=0.0625)), 'logit_scale'),
    ):
        with pytest.raises(RuntimeError, match=msg):
            ops.lm_head_weight(bad)


def test_device_lens_is_list_like_without_touching_the_device_until_asked():
    from align_anything_b200 import ops

    host = ops.as_device_lens.__wrapped__ if hasattr(ops.as_device_lens, '__wrapped__') else None
    assert host is None
    dl = ops.DeviceLens(torch.tensor([3, 0, 7], dtype=torch.int32), 9)  # a CPU tensor stands in for the device one here
    assert dl.bound == 9 and len(dl) == 3 and dl._host is None
    assert list(dl) == [3, 0, 7] and dl[2] == 7 and dl == [3, 0, 7] and dl._host == [3, 0, 7]


def test_dense_actor_plan_layout():
    """ops._dense_actor_plan (the text PPO actor node on K1f, trainers/text_to_text/ppo.py:336-349): sample b scores the rows
    [start, L - 1) of its (L, V) tile against ids[b, start + 1 :]; one segment per sample, the gradient tile is (B * L, V)."""
    from align_anything_b200 import ops

    B, L_, start, V = 3, 12, 4, 100
    plan = ops._dense_actor_plan(B, L_, start, L_ * V, V, L_, 'cpu')
    W = L_ - 1 - start
    t = plan.dev
    assert plan.n_seg == B and plan.n_rows == B * W and plan.out_shape == (B, W) and plan.n_tile_rows == B * L_
    assert t[0, :B].tolist() == [b * L_ * V + start * V for b in range(B)]     # logits element offsets
    assert t[1, :B].tolist() == [b * L_ + start + 1 for b in range(B)]          # label offsets: next token
    assert t[2, :B].tolist() == [b * W for b in range(B)]                       # output offsets
    assert t[3].tolist() == [b * W for b in range(B + 1)]                       # prefix row counts
    assert t[4, :B].tolist() == [b * L_ + start for b in range(B)]              # first scored row in the gradient tile
    assert plan.n_tile_rows % plan.n_seg == 0                                   # what aa_logprob_actor_fused requires


def _k1f_slot(scored: bool, i: int, z: int, G: int, S: int, Z: int) -> int:
    """The work-list position fused_actor_prep_kernel (csrc/logprob_fused.cu) gives a row when the list alternates G scored
    rows and G zero rows: i = flat index of a scored row, z = index of a zero row in tile order, S / Z = their totals."""
    if scored:
        return i + min((i // G) * G, Z)              # zero rows of the earlier rounds come first
    return min((z // G + 1) * G, S) + z              # scored rows of this and the earlier rounds come first


def test_k1f_interleaved_work_list_is_a_permutation():
    """The interleaved order must place every row exactly once in [0, S + Z), for any grid size and any split between scored
    and zero rows, and while both kinds last every CTA (static stride G) must alternate scored / zero rows."""
    import random

    rng = random.Random(5)
    cases = [(148, 8695, 7721), (102, 66, 36), (80, 36, 44), (1, 5, 3), (7, 0, 9), (7, 9, 0), (148, 100, 20000), (296, 20000, 3)]
    cases += [(rng.randint(1, 300), rng.randint(0, 3000), rng.randint(0, 3000)) for _ in range(40)]
    for G, S, Z in cases:
        slots = [_k1f_slot(True, i, 0, G, S, Z) for i in range(S)] + [_k1f_slot(False, 0, z, G, S, Z) for z in range(Z)]
        assert sorted(slots) == list(range(S + Z)), (G, S, Z)
        kind = [None] * (S + Z)
        for i in range(S):
            kind[_k1f_slot(True, i, 0, G, S, Z)] = 'S'
        for z in range(Z):
            kind[_k1f_slot(False, 0, z, G, S, Z)] = 'Z'
        full_rounds = min(S, Z) // G  # rounds in which both kinds fill a whole block of G
        for cta in range(min(G, S + Z)):
            mine = kind[cta::G][: 2 * full_rounds]
            assert mine == ['S', 'Z'] * full_rounds, (G, S, Z, cta)


def test_single_pass_routing(monkeypatch):
    """ops._single_pass_ok: K1f's tile is written for an upstream gradient of 1, so fp16 logits (loss scaling) stay on the
    two-pass path unless ops._FUSED_F16 is set, and so do rows shorter than ops._FUSED_MIN_ROW_BYTES (192 KB by default:
    K1f measured 0.83x of the two-pass path at V = 32064 bf16, 1.15x at 128256, 1.25x at 152064), a node whose knob is
    off, and logits that need no gradient."""
    from align_anything_b200 import ops

    def tile(V, dtype):
        return torch.empty((1, 1, V), dtype=dtype)

    assert ops._FUSED_MIN_ROW_BYTES == 192 * 1024 and not ops._FUSED_F16
    assert ops._single_pass_ok(tile(152064, torch.bfloat16)) and ops._single_pass_ok(tile(128257, torch.bfloat16))
    assert not ops._single_pass_ok(tile(152064, torch.bfloat16), enabled=False)
    assert not ops._single_pass_ok(tile(152064, torch.bfloat16), needs_grad=False)
    assert not ops._single_pass_ok(tile(32064, torch.bfloat16)) and not ops._single_pass_ok(tile(65536, torch.bfloat16))
    assert ops._single_pass_ok(tile(65536, torch.float32))            # 256 KB rows
    assert not ops._single_pass_ok(tile(152064, torch.float16))       # fp16: loss scaling
    monkeypatch.setattr(ops, '_FUSED_F16', True)
    assert ops._single_pass_ok(tile(152064, torch.float16)) and not ops._single_pass_ok(tile(32064, torch.float16))
    monkeypatch.setattr(ops, '_FUSED_MIN_ROW_BYTES', 0)
    assert ops._single_pass_ok(tile(523, torch.bfloat16)) and ops._single_pass_ok(tile(523, torch.float16))
