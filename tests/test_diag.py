"""PPO update diagnostics (DESIGN.md §9n) without a device: the metrics on hand-made accumulator rows, the merge of
rows by each column's rule, the column list against the header, the tensor-to-group map, the stop rule, the drivers'
argument errors, the library's exports, and two gloo ranks merging their rows to one decision."""
import os
import re
import socket

import numpy as np
import pytest
import torch

import diag_ref
from rl_collision_avoidance_b200.model import diagnostics as D
from rl_collision_avoidance_b200.model.net import TENSORS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def row(**cols):
    r = D.EMPTY_ROW.copy()
    for k, v in cols.items():
        r[D.COL[k]] = v
    return r


def critic_row(t, v):
    t, v = np.asarray(t, dtype=np.float64), np.asarray(v, dtype=np.float64)
    return row(n=len(t), sum_err=(t - v).sum(), sum_err_sq=((t - v) ** 2).sum(), sum_target=t.sum(),
               sum_target_sq=(t * t).sum(), sum_value=v.sum())


def header_defines():
    src = open(os.path.join(ROOT, 'include', 'rlca.h')).read()
    return {k: int(v) for k, v in re.findall(r'#define (RLCA_\w+) (\d+)\b', src)}


def test_column_list_matches_the_header():
    h = header_defines()
    assert len(D.COLUMNS) == h['RLCA_PPO_DIAG_COLUMNS']
    assert len(set(D.NAMES)) == len(D.NAMES)
    for name, define in (('n', 'N'), ('sum_kl', 'SUM_KL'), ('sum_kl_k3', 'SUM_KL_K3'), ('clipped', 'CLIPPED'),
                         ('cut', 'CUT'), ('sum_ratio', 'SUM_RATIO'), ('sum_err', 'SUM_ERR'),
                         ('sum_target', 'SUM_TARGET'), ('sum_value', 'SUM_VALUE'), ('sum_adv', 'SUM_ADV'),
                         ('mean_out_0', 'MEAN_OUT'), ('action_out_0', 'ACTION_OUT'), ('max_ratio', 'MAX_RATIO'),
                         ('min_ratio', 'MIN_RATIO'), ('grad_steps', 'GRAD_STEPS'),
                         ('grad_sumsq.logstd', 'GRAD_SUMSQ'), ('max_grad_sumsq', 'MAX_GRAD_SUMSQ')):
        assert D.COL[name] == h['RLCA_PPO_DIAG_' + define], name
    assert h['RLCA_PPO_DIAG_MAX_GRAD_SUMSQ'] - h['RLCA_PPO_DIAG_GRAD_SUMSQ'] == h['RLCA_POLICY_NTENSORS'] == len(TENSORS)
    assert [r for r in D.RULES if r != 'sum'] == ['max', 'min', 'max']
    assert set(diag_ref.SUM_COLUMNS) | {'max_ratio', 'min_ratio'} == set(D.NAMES[:D.COL['grad_steps']])


def test_every_tensor_is_in_one_group():
    groups = [D.tensor_group(name) for name, _ in TENSORS]
    assert len(groups) == 23 and set(groups) == set(D.GROUPS)
    count = {g: groups.count(g) for g in D.GROUPS}
    assert count == {'actor_conv': 4, 'critic_conv': 4, 'actor_fc': 4, 'critic_fc': 4, 'heads': 6, 'logstd': 1}
    assert D.tensor_group('crt_fea_cv2.bias') == 'critic_conv' and D.tensor_group('act_fc1.weight') == 'actor_fc'
    assert D.tensor_group('critic.weight') == 'heads'


def test_explained_variance_one_zero_negative_nan():
    t = np.array([1.0, 2.0, 4.0, -3.0])
    ev = lambda v: D.metrics(critic_row(t, v))['explained_variance']
    assert ev(t) == pytest.approx(1.0)
    assert ev(t + 5.0) == pytest.approx(1.0)                    # a constant bias leaves the variance explained ...
    assert D.metrics(critic_row(t, t + 5.0))['value_bias'] == pytest.approx(5.0)      # ... and shows here
    assert ev(np.full(4, 7.0)) == pytest.approx(0.0)            # a constant critic explains nothing
    assert ev(-t) == pytest.approx(-3.0)                        # Var(2 t) / Var(t) = 4
    assert np.isnan(D.metrics(critic_row(np.full(4, 2.5), t))['explained_variance'])
    assert np.isnan(D.metrics(critic_row(np.full(1000, 0.1), np.zeros(1000)))['explained_variance'])
    m = D.metrics(critic_row(t, t - 1.0))
    assert m['value_rmse'] == pytest.approx(1.0) and m['value_bias'] == pytest.approx(-1.0)


def test_fractions_ratio_and_saturation():
    m = D.metrics(row(n=8, clipped=2, cut=1, sum_ratio=8.8, max_ratio=1.5, min_ratio=0.7, sum_kl=0.4, sum_kl_k3=0.08,
                      mean_out_0=0, mean_out_1=4, action_out_0=8, action_out_1=2, sum_adv=4.0, sum_adv_sq=10.0))
    assert m['clip_fraction'] == 0.25 and m['cut_fraction'] == 0.125
    assert m['ratio_mean'] == pytest.approx(1.1) and (m['ratio_max'], m['ratio_min']) == (1.5, 0.7)
    assert m['approx_kl'] == pytest.approx(0.05) and m['approx_kl_k3'] == pytest.approx(0.01)
    assert m['mean_saturation'] == [0.0, 0.5] and m['action_saturation'] == [1.0, 0.25]
    assert m['adv_mean'] == 0.5 and m['adv_std'] == pytest.approx(1.0)


def test_gradient_norms():
    cols = {'grad_sumsq.' + name: 0.0 for name, _ in TENSORS}
    cols.update({'grad_sumsq.logstd': 2.0, 'grad_sumsq.act_fea_cv1.weight': 8.0, 'grad_sumsq.act_fea_cv2.bias': 10.0,
                 'grad_sumsq.crt_fc2.weight': 32.0, 'grad_sumsq.actor2.bias': 1.0, 'grad_sumsq.critic.weight': 17.0})
    m = D.metrics(row(grad_steps=2, max_grad_sumsq=49.0, **cols))
    assert m['grad_norm'] == pytest.approx(np.sqrt(70.0 / 2)) and m['grad_norm_max'] == 7.0
    assert m['grad_norm_by_group'] == pytest.approx({'actor_conv': 3.0, 'critic_conv': 0.0, 'actor_fc': 0.0,
                                                     'critic_fc': 4.0, 'heads': 3.0, 'logstd': 1.0})


def test_metrics_match_the_reference_on_a_batch():
    b = diag_ref.decisive_batch(np.random.RandomState(5), 300)
    cols, _ = diag_ref.ref_row(b)
    m, ref = D.metrics(row(**cols)), diag_ref.ref_metrics(cols)
    for k, v in ref.items():
        assert m[k] == pytest.approx(v, rel=1e-12, abs=1e-12), k
    assert 0 < m['clip_fraction'] < 1 and 0 < m['cut_fraction'] < m['clip_fraction']
    assert m['approx_kl_k3'] > 0 and all(0 < x < 1 for x in m['mean_saturation'] + m['action_saturation'])


def test_rows_merge_by_their_rule_and_an_empty_epoch_is_nan():
    a = row(n=3, sum_ratio=3.3, max_ratio=1.4, min_ratio=0.9, grad_steps=1, max_grad_sumsq=4.0)
    b = row(n=5, sum_ratio=4.5, max_ratio=1.2, min_ratio=0.6, grad_steps=2, max_grad_sumsq=9.0)
    merged = D.merge_rows([a, b, D.EMPTY_ROW])
    assert merged[D.COL['n']] == 8 and merged[D.COL['sum_ratio']] == pytest.approx(7.8)
    assert merged[D.COL['max_ratio']] == 1.4 and merged[D.COL['min_ratio']] == 0.6
    assert merged[D.COL['grad_steps']] == 3 and merged[D.COL['max_grad_sumsq']] == 9.0
    assert np.array_equal(D.merge_rows([]), D.EMPTY_ROW)
    m = D.metrics(np.stack([a, D.EMPTY_ROW]))
    assert m['rows'] == 3 and m['ratio_mean'] == pytest.approx(1.1) and m['ratio_max'] == 1.4
    assert [e['rows'] for e in m['per_epoch']] == [3, 0]
    empty = m['per_epoch'][1]
    for k in ('approx_kl', 'approx_kl_k3', 'clip_fraction', 'ratio_mean', 'ratio_max', 'ratio_min', 'explained_variance',
              'value_rmse', 'adv_std', 'grad_norm', 'grad_norm_max'):
        assert np.isnan(empty[k]), k
    line = D.format_line(7, dict(m, epochs_run=1, logstd=[0.0, -0.5]))
    assert line.startswith('update 7, epochs 1, rows 3, ') and '\n' not in line


def test_stop_rule():
    assert D.over_target_kl(row(n=10, sum_kl_k3=0.31), 0.03)
    assert not D.over_target_kl(row(n=10, sum_kl_k3=0.29), 0.03)
    assert not D.over_target_kl(row(n=10, sum_kl_k3=0.3), 0.03 + 1e-12)
    assert D.over_target_kl(row(n=10, sum_kl_k3=float('nan')), 0.03)      # a policy that blew up stops the update
    assert not D.over_target_kl(D.EMPTY_ROW, 0.03)                        # an epoch without rows does not
    for bad in (0, -1, float('nan'), float('inf')):
        with pytest.raises(ValueError):
            D.check_target_kl(bad)
    assert D.check_target_kl('0.02') == 0.02


@pytest.mark.parametrize('stage', [1, 2])
@pytest.mark.parametrize('value', ['0', 'nan', '-1', 'inf'])
def test_drivers_reject_a_bad_target_kl(capsys, monkeypatch, stage, value):
    def fail(*a, **k):
        raise AssertionError('device work before the argument checks')
    monkeypatch.setattr(torch.cuda, 'set_device', fail)
    import ppo_stage1
    import ppo_stage2
    kw = {} if stage == 1 else dict(stage=2, world_cls=ppo_stage2.StageWorld, num_env=ppo_stage2.NUM_ENV,
                                    batch_size=ppo_stage2.BATCH_SIZE, epoch=ppo_stage2.EPOCH, ckpt='stage2.pth')
    with pytest.raises(SystemExit) as e:
        ppo_stage1.main(argv=['--target-kl=' + value], **kw)
    assert e.value.code == 2
    assert '--target-kl: the target KL must be finite and > 0' in capsys.readouterr().err


def test_target_kl_implies_diagnostics(monkeypatch):
    """--target-kl alone opens diag.log, as --diagnostics does; neither flag leaves it alone."""
    import ppo_stage1

    class Reached(Exception):
        pass

    def reached(*a, **k):
        raise Reached

    def no_env(*a, **k):
        raise RuntimeError('past the loggers')
    monkeypatch.setattr(torch.cuda, 'set_device', lambda *a, **k: None)
    monkeypatch.setattr(ppo_stage1, 'make_loggers', lambda: (None, None))
    monkeypatch.setattr(ppo_stage1, 'setup_diag_log', reached)
    for argv in (['--target-kl', '0.02'], ['--diagnostics']):
        with pytest.raises(Reached):
            ppo_stage1.main(argv=argv, world_cls=no_env)
    with pytest.raises(RuntimeError, match='past the loggers'):
        ppo_stage1.main(argv=[], world_cls=no_env)


def test_library_exports_the_new_entries(built):
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    for name in ('rlca_ppo_diag_accumulate', 'rlca_grad_sumsq'):
        assert hasattr(lib, name) and name in _lib.SYMBOLS
    # argument errors are reported before any device work
    assert lib.rlca_grad_sumsq(None, None, None, None) == 1 and b'NULL' in lib.rlca_last_error()
    assert lib.rlca_ppo_diag_accumulate(None, None, None, None, None, None, None, None, 4, 0.1, None, None, None) == 1


# ------------------------------------------------------------------------------------------------ two gloo ranks
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_rows(rank):
    """Two epochs of a rank: rank 0 moved little, rank 1 far; only the merged row of epoch 0 is over the target."""
    rs = np.random.RandomState(10 + rank)
    rows = []
    for epoch in range(2):
        b = diag_ref.decisive_batch(rs, (40, 25)[rank], spread=(0.02, 0.6)[rank] if epoch == 0 else 0.01)
        cols, _ = diag_ref.ref_row(b)
        rows.append(row(grad_steps=1 + rank, max_grad_sumsq=3.0 + rank, **cols))
    return np.stack(rows)


TARGET = 0.01


def _merge_worker(rank, world_size, port, out):
    import torch.distributed as dist
    from rl_collision_avoidance_b200.parallel import allreduce_diagnostics
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world_size)
    try:
        local = _rank_rows(rank)
        acc = torch.from_numpy(local.copy())
        one = allreduce_diagnostics(acc[0].clone(), D.RULES)          # the epoch-boundary merge of one row
        allreduce_diagnostics(acc, D.RULES)                           # the end-of-update merge of all rows
        out.put((rank, acc.numpy(), one.numpy(), D.over_target_kl(local[0], TARGET),
                 [D.over_target_kl(r, TARGET) for r in acc.numpy()]))
    finally:
        dist.destroy_process_group()


def test_two_ranks_merge_to_the_same_row_and_decision():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_merge_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    locals_ = [_rank_rows(r) for r in range(2)]
    want = np.stack([D.merge_rows([locals_[0][e], locals_[1][e]]) for e in range(2)])
    for rank, acc, one, local_stop, stops in res:
        assert np.allclose(acc, want, rtol=1e-15, atol=0) and np.array_equal(acc[:, D.COL['n']], [65, 65])
        assert np.array_equal(acc[:, D.COL['max_ratio']], want[:, D.COL['max_ratio']])
        assert np.array_equal(acc[:, D.COL['min_ratio']], want[:, D.COL['min_ratio']])
        assert np.array_equal(one, acc[0])
        assert stops == [True, False]
    assert np.array_equal(res[0][1], res[1][1])                       # bit for bit the same rows on both ranks
    assert [r[3] for r in res] == [False, True]                       # alone, the ranks would have disagreed
