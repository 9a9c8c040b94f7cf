"""The SL-policy on the device (DESIGN.md §9g): the behaviour-cloning loss and gradient against float64 autograd,
demonstration recording against the recording rule rebuilt in torch, supervised training, and the driver end to end."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from golden_inputs import synthetic_state_dict
from test_learner_shapes_gpu import Checks, decisive_pool, grad_views, layer_scale, make_policy, maxabs, params64, \
    ref_forward

pytestmark = pytest.mark.gpu

BC_NB = [1, 67, 129, 512, 1024, 1793]
MODES = {1: 'tc', 2: 'fc1tc', 0: 'fp32'}
CRITIC = ('crt_', 'critic.')


def _bits(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------ loss and gradient
@pytest.fixture(scope='module')
def bc_pool(built):
    p = decisive_pool(max(BC_NB))
    p['target'] = np.stack([np.clip(p['act'][:, 0], 0, 1), np.clip(p['act'][:, 1], -1, 1)], 1).astype(np.float32)
    return p


def ref_bc(pool, nb):
    P = params64(synthetic_state_dict(), grad=True)
    d64 = lambda k: torch.from_numpy(np.ascontiguousarray(pool[k][:nb])).cuda().double()
    _, mean, _ = ref_forward(P, d64('obs'), d64('gs'))
    loss = ((mean - d64('target')) ** 2).sum(1).mean()
    loss.backward()
    return float(loss.detach()), {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in P.items()}


@pytest.mark.parametrize('mode', list(MODES), ids=list(MODES.values()))
@pytest.mark.parametrize('nb', BC_NB, ids=[f'nb{n}' for n in BC_NB])
def test_bc_loss_and_gradient_vs_float64_autograd(bc_pool, nb, mode):
    """BC loss + rlca_policy_backward: the loss to 1e-5 relative, every actor gradient to 5e-5 of its layer's scale
    (DESIGN.md §8's bound), and the logstd and critic gradients exactly 0."""
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.net import _ptr
    pol = make_policy(nb, mode)
    cu = lambda k: torch.from_numpy(np.ascontiguousarray(bc_pool[k][:nb])).cuda()
    obs, gs, target = cu('obs').reshape(nb, 1536).contiguous(), cu('gs'), cu('target')
    lib, ws, st = pol.lib, pol._workspace(nb), pol._stream()
    v, mean, loss = torch.empty(nb, device='cuda'), torch.empty(nb, 2, device='cuda'), torch.zeros(1, device='cuda')
    pol.grad.fill_(1.0)
    _lib.check(lib.rlca_policy_forward(ws, _ptr(pol.flat), _ptr(obs), _ptr(gs), nb, _ptr(v), _ptr(mean), st))
    _lib.check(lib.rlca_bc_loss_fwd_bwd(ws, _ptr(pol.flat), _ptr(mean), _ptr(target), nb, _ptr(loss), st))
    _lib.check(lib.rlca_policy_backward(ws, _ptr(pol.flat), _ptr(obs), _ptr(gs), nb, _ptr(pol.grad), st))
    torch.cuda.synchronize()
    ref_loss, ref_grads = ref_bc(bc_pool, nb)
    what = f'bc nb={nb} {MODES[mode]}'
    check = Checks()
    check(f'{what} loss', abs(float(loss[0]) - ref_loss), 1e-5 * abs(ref_loss))
    views = grad_views(pol, pol.grad)
    for name, r in ref_grads.items():
        if name == 'logstd' or name.startswith(CRITIC):
            check(f'{what} grad {name} (exactly 0)', maxabs(views[name].double()), 0.0)
        else:
            check(f'{what} grad {name}', maxabs(views[name].double() - r), 5e-5 * layer_scale(ref_grads, name))
    check.done()


def test_bc_loss_rejects_bad_arguments(built):
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.model.net import _ptr
    pol = make_policy(8)
    ws, m, loss = pol._workspace(8), torch.zeros(9, 2, device='cuda'), torch.zeros(1, device='cuda')
    for args in ((ws, _ptr(pol.flat), _ptr(m), _ptr(m), 9, _ptr(loss)), (ws, _ptr(pol.flat), _ptr(m), _ptr(m), 0, _ptr(loss)),
                 (ws, _ptr(pol.flat), None, _ptr(m), 4, _ptr(loss)), (None, _ptr(pol.flat), _ptr(m), _ptr(m), 4, _ptr(loss))):
        assert pol.lib.rlca_bc_loss_fwd_bwd(*args, pol._stream()) == 1


# ------------------------------------------------------------------------------------------------ recording
def clip_action(a, cfg):
    """The tick's clip (rlca_physics_kernel): |x| > 3e38 or NaN -> 0, then the action box."""
    a = torch.where(a.abs() <= 3.0e38, a, torch.zeros_like(a))
    return torch.stack((a[:, 0].clamp(cfg.v_min, cfg.v_max), a[:, 1].clamp(cfg.w_min, cfg.w_max)), 1)


def drive(env, ctrl, ticks, demos, action_hook=None):
    """evaluate()'s loop with the controller, appending to every DemoSet of `demos` before each tick, and the rows the
    recording rule expects, rebuilt in torch from the tick's stack, gs, action, meta and previous flags."""
    N, dev = env.N, env.device
    circle = int(env.cfg.auto_reset) == 0
    env.reset_world()
    env.reset_pose()
    env.generate_goal_point()
    obs = env.get_laser_observation()
    stacks = [obs[:, None, :].repeat(1, 3, 1).contiguous(), torch.empty(N, 3, env.beam_mum, device=dev)]
    terminal = torch.zeros(N, dtype=torch.bool, device=dev)
    rows, skipped = {'obs': [], 'gs': [], 'action': []}, []
    for tick in range(ticks):
        k = tick & 1
        action = ctrl()
        if action_hook is not None:
            action = action_hook(tick, action)
        if env.cfg.auto_reset == 2:
            rec = env.state['meta'][:, 3] == 0
        elif circle:
            rec = ~terminal
        else:
            rec = torch.ones(N, dtype=torch.bool, device=dev)
        skipped.append(int((~rec).sum()))
        rows['obs'].append(stacks[k].reshape(N, -1)[rec].clone())
        rows['gs'].append(env.gs[rec].clone())
        rows['action'].append(clip_action(action, env.cfg)[rec])
        for d in demos:
            d.append(action, stacks[k], env.flags if circle and tick > 0 else None)
        scaled = torch.stack((torch.where(terminal, 0.0, action[:, 0]), action[:, 1]), 1) if circle else action
        env.control_vel(scaled, stack_in=stacks[k], stack_out=stacks[1 - k])
        if circle:
            terminal = env.flags[:, 0] != 0
    return {key: torch.cat(v) for key, v in rows.items()}, skipped


def assert_rows_equal(got, want, n):
    """got: (obs, gs, action) of a DemoSet or collect(); want: the expected rows; the first n of them, bit for bit"""
    assert got[0].shape[0] == n, (got[0].shape[0], n)
    for g, key in zip(got, ('obs', 'gs', 'action')):
        assert torch.equal(_bits(g), _bits(want[key][:n])), key


def make_env(name, worlds, seed=3):
    from rl_collision_avoidance_b200.evaluation import AUTO_RESET
    from rl_collision_avoidance_b200.orca import NhOrcaController
    from rl_collision_avoidance_b200.stage_world import StageWorld
    env = StageWorld(512, scenario=name, num_worlds=worlds, seed=seed, auto_reset=AUTO_RESET[name])
    return env, NhOrcaController(env, obstacles=True)


@pytest.mark.parametrize('name, worlds, ticks', [('stage1', 171, 24), ('stage2', 8, 160), ('circle', 4, 420)])
def test_recording_equals_the_rule(built, name, worlds, ticks):
    """Every row of the device dataset equals the row the recording rule gives, in order, with the same count; a
    dataset smaller than one tick keeps the first `capacity` rows; collect() records the same rows."""
    from rl_collision_avoidance_b200.sl import DemoSet, collect
    env, ctrl = make_env(name, worlds)
    small = 1000 if name == 'stage1' else 37
    big_cap = env.N * ticks
    demos = [DemoSet(env, big_cap), DemoSet(env, small)]
    want, skipped = drive(env, ctrl, ticks, demos)
    total = want['obs'].shape[0]
    print(f'[recording] {name}: {env.N} agents x {ticks} ticks, {total} rows, skipped agent-ticks {sum(skipped)}')
    if name == 'stage1':
        assert total == env.N * ticks and small < env.N
    else:                   # the rule had something to skip, and agents that were recorded on the same tick
        assert any(0 < s < env.N for s in skipped), skipped
    assert_rows_equal(demos[0].rows(), want, total)
    assert_rows_equal(demos[1].rows(), want, small)
    part = total - env.N // 2                         # collect() stops once its dataset is full
    assert_rows_equal(collect(env, ctrl, part), want, part)


def test_recording_clips_like_the_tick(built):
    """Raw actions outside the box, infinite, NaN or beyond 3e38 are stored as the tick applies them."""
    from rl_collision_avoidance_b200.sl import DemoSet
    env, ctrl = make_env('stage1', 2)
    bad = torch.tensor([[1.5, -2.0], [-0.5, 3.0], [math.inf, -math.inf], [math.nan, 0.5], [3.2e38, -3.2e38],
                        [0.25, -0.75]], device='cuda')

    def hook(tick, action):
        a = action.clone()
        a[:bad.shape[0]] = bad
        return a
    demo = DemoSet(env, env.N * 3)
    want, _ = drive(env, ctrl, 3, [demo], action_hook=hook)
    assert_rows_equal(demo.rows(), want, env.N * 3)
    assert demo.action[:6].tolist() == [[1.0, -1.0], [0.0, 1.0], [0.0, 0.0], [0.0, 0.5], [0.0, 0.0], [0.25, -0.75]]


def test_recording_rejects_bad_arguments(built):
    from rl_collision_avoidance_b200 import _lib
    from rl_collision_avoidance_b200.sl import DemoSet
    from rl_collision_avoidance_b200.model.net import _ptr
    env, ctrl = make_env('stage1', 1)
    demo = DemoSet(env, 100)
    a = ctrl()
    stack = torch.zeros(env.N, 3, 512, device='cuda')
    st = C.byref(env._state_struct(env._cur))

    def call(io=None, cfg=None, demo_set=None):
        io = io or _lib.StepIO(_ptr(a), None, None, None, None, _ptr(env.gs), None, _ptr(stack), None)
        return env.lib.rlca_demo_append(C.byref(cfg or env.cfg), st, C.byref(io), C.byref(demo_set or demo._set),
                                        env._stream())
    assert call() == 0
    live = torch.ones(env.N, dtype=torch.uint8, device='cuda')
    assert call(io=_lib.StepIO(_ptr(a), _ptr(live), None, None, None, _ptr(env.gs), None, _ptr(stack), None)) == 3
    assert call(io=_lib.StepIO(_ptr(a), None, None, None, None, _ptr(env.gs), None, None, None)) == 1
    flat = torch.zeros(env.N * 1536 + 4, device='cuda')
    assert call(io=_lib.StepIO(_ptr(a), None, None, None, None, _ptr(env.gs), None, _ptr(flat[1:]), None)) == 1
    s = demo._set
    assert call(demo_set=_lib.DemoSet(s.obs_dev, s.gs_dev, s.action_dev, s.count_dev, 0)) == 1
    assert call(demo_set=_lib.DemoSet(s.obs_dev, s.gs_dev, s.action_dev, None, 100)) == 1
    cfg = _lib.EnvConfig.from_buffer_copy(env.cfg)
    cfg.auto_reset = 3
    assert call(cfg=cfg) == 1
    cfg = _lib.EnvConfig.from_buffer_copy(env.cfg)
    cfg.beams = 510
    assert call(cfg=cfg) == 3
    with pytest.raises(ValueError):
        DemoSet(env, 0)
    torch.cuda.synchronize()
    assert demo.count() == env.N                      # the one good call


# ------------------------------------------------------------------------------------------------ training
TRAIN_LR, TRAIN_BATCH, TRAIN_EPOCHS = 3e-4, 256, 10
# measured on an H100: the held-out loss after 10 epochs (280 steps) is 0.126 of its initial value (0.611 -> 0.077)
HELD_OUT_FACTOR = 0.25


@pytest.fixture(scope='module')
def stage1_rows(built):
    from rl_collision_avoidance_b200.sl import collect
    env, ctrl = make_env('stage1', 8, seed=11)
    data = collect(env, ctrl, 8000)
    assert data[0].shape[0] == 8000
    return data


def train(data, seed=0):
    from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy
    from rl_collision_avoidance_b200.sl import sl_loss, sl_update
    g = torch.Generator(device='cpu')
    g.manual_seed(seed)
    perm = torch.randperm(data[0].shape[0], generator=g).cuda()
    held, rows = perm[:1000], perm[1000:]
    pol = CNNPolicy(frames=3, action_space=2, seed=seed, max_batch=TRAIN_BATCH)
    init = pol.flat.clone()
    opt = Adam(pol.parameters(), lr=TRAIN_LR)
    gen = torch.Generator(device='cuda')
    gen.manual_seed(seed)
    before = sl_loss(pol, data, TRAIN_BATCH, rows=held)
    losses = sl_update(pol, opt, data, TRAIN_BATCH, TRAIN_EPOCHS, generator=gen, rows=rows)
    after = sl_loss(pol, data, TRAIN_BATCH, rows=held)
    return pol, init, before, after, losses


def test_training_lowers_the_held_out_loss_deterministically(stage1_rows):
    from rl_collision_avoidance_b200.model.net import TENSORS
    pol, init, before, after, losses = train(stage1_rows)
    print(f'[training] held-out loss {before:.6f} -> {after:.6f} (x {after / before:.3f}), '
          f'{len(losses)} steps, first / last minibatch loss {losses[0]:.6f} / {losses[-1]:.6f}')
    assert len(losses) == TRAIN_EPOCHS * math.ceil(7000 / TRAIN_BATCH)
    assert after < HELD_OUT_FACTOR * before, (before, after)
    for i, (name, _) in enumerate(TENSORS):
        lo, hi = pol.offsets[i], pol.offsets[i + 1]
        same = torch.equal(_bits(pol.flat[lo:hi]), _bits(init[lo:hi]))
        if name == 'logstd' or name.startswith(CRITIC):
            assert same, f'{name} changed'
        else:
            assert not same, f'{name} did not change'
    pol2, _, before2, after2, losses2 = train(stage1_rows)
    assert torch.equal(_bits(pol.flat), _bits(pol2.flat))
    assert (before, after, losses) == (before2, after2, losses2)


# ------------------------------------------------------------------------------------------------ driver
def test_sl_train_then_evaluate_end_to_end(built, tmp_path, capsys):
    import evaluate
    import sl_train
    out = tmp_path / 'sl.pth'
    sl_train.main(['--scenario', 'stage1', '--samples', '2000', '--num-worlds', '2', '--epochs', '2',
                   '--batch-size', '256', '--out', str(out)])
    text = capsys.readouterr().out
    assert 'epoch 2  train loss' in text and 'held-out loss' in text and out.exists(), text
    evaluate.main(['--scenario', 'stage1', '--policy', str(out), '--num-worlds', '1', '--episodes', '1'])
    text = capsys.readouterr().out
    assert 'stage1  robots 24' in text and 'success' in text, text
