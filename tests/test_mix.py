"""Training on a mix of scenarios (DESIGN.md §9l), without a device: every command-line rejection of ppo_stage2.py's and
ppo_stage1.py's main before any device work, the --mix parser, the column ranges and per-rank world offsets of a mix,
and the alignment check of a component's rollout slices."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _trainer(stage):
    import ppo_stage1
    if stage == 1:
        return lambda argv: ppo_stage1.main(argv=argv)
    import ppo_stage2
    return lambda argv: ppo_stage1.main(stage=2, world_cls=ppo_stage2.StageWorld, num_env=ppo_stage2.NUM_ENV,
                                        batch_size=ppo_stage2.BATCH_SIZE, epoch=ppo_stage2.EPOCH, ckpt='stage2.pth',
                                        argv=argv)


@pytest.fixture
def no_device(monkeypatch):
    """Any device work after the argument checks fails the test at once."""
    def fail(*a, **k):
        raise AssertionError('device work before the argument checks')
    monkeypatch.setattr(torch.cuda, 'set_device', fail)


MIX = 'stage2:2,random:3,circle:1'


@pytest.mark.parametrize('argv, message', [
    (['--mix', MIX, '--scenario', 'stage2'], '--mix gives the scenarios and their world counts'),
    (['--mix', MIX, '--scenario', 'random'], '--mix gives the scenarios and their world counts'),
    (['--mix', MIX, '--num-worlds', '4'], '--mix gives the scenarios and their world counts'),
    (['--mix', 'stage2:2,maze:3'], "unknown scenario 'maze'"),
    (['--mix', 'stage2:2,stage2:3'], 'stage2 appears more than once'),
    (['--mix', 'random:2,circle:1,random:1'], 'random appears more than once'),
    (['--mix', 'stage2:0'], 'stage2 needs at least 1 world, got 0'),
    (['--mix', 'circle:-3'], 'circle needs at least 1 world, got -3'),
    (['--mix', 'stage2:two'], 'the world count of stage2 must be an integer'),
    (['--mix', 'stage2'], '--mix entries are name:worlds'),
    (['--mix', 'stage2:2,'], '--mix entries are name:worlds'),
    (['--mix', 'stage1:2,stage2:2'], 'stage 1 cannot be mixed'),
    (['--mix', 'stage2:2,circle:1', '--random-robots', '16'],
     'apply to --scenario random or a random component of --mix only'),
    (['--mix', 'stage2:2', '--random-timeout', '100'], 'apply to --scenario random or a random component of --mix only'),
    (['--mix', 'random:2', '--random-robots', '1'], 'robots_per_world must be in 2..64'),
    (['--mix', 'random:2', '--random-timeout', '0'], '--random-timeout must be >= 1'),
])
def test_stage2_cli_rejects_bad_mix(capsys, no_device, argv, message):
    with pytest.raises(SystemExit) as e:
        _trainer(2)(argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


@pytest.mark.parametrize('argv', [['--mix', MIX], ['--mix', 'stage2:2'], ['--mix', 'stage1:1']])
def test_stage1_cli_rejects_mix(capsys, no_device, argv):
    with pytest.raises(SystemExit) as e:
        _trainer(1)(argv)
    assert e.value.code == 2
    assert '--mix trains with ppo_stage2.py' in capsys.readouterr().err


def test_random_flags_are_accepted_with_a_random_component(monkeypatch):
    """Every --random-* flag passes the checks with a random component: main reaches the device (here a sentinel)."""
    class Reached(Exception):
        pass

    def reached(*a, **k):
        raise Reached
    monkeypatch.setattr(torch.cuda, 'set_device', reached)
    with pytest.raises(Reached):
        _trainer(2)(['--mix', 'stage2:1,random:2', '--random-robots', '16', '--random-side', '8',
                     '--random-separation', '1.2', '--random-min-travel', '3', '--random-timeout', '300'])


def test_parse_mix_keeps_the_order_given():
    from rl_collision_avoidance_b200.mix import parse_mix
    assert parse_mix('stage2:31,random:128,circle:14') == [('stage2', 31), ('random', 128), ('circle', 14)]
    assert parse_mix('circle:1, Random:2') == [('circle', 1), ('random', 2)]
    assert parse_mix('random:5') == [('random', 5)]


def test_column_ranges_and_world_offsets():
    """--mix stage2:31,random:128,circle:14 --random-robots 16: 31 x 44 + 128 x 16 + 14 x 50 = 4112 columns in the
    order given; rank r starts component k at world r * W_k, as a single-scenario run of W_k worlds per GPU."""
    import ppo_stage1
    from rl_collision_avoidance_b200.mix import parse_mix
    from rl_collision_avoidance_b200.scenarios import make_scenario
    mix = parse_mix('stage2:31,random:128,circle:14')
    sc = make_scenario('random', robots_per_world=16)
    for rank in range(4):
        comps = ppo_stage1.mix_components(mix, sc, rank)
        assert [c.name for c in comps] == ['stage2', 'random', 'circle']
        assert [c.robots_per_world for c in comps] == [44, 16, 50]
        assert [c.cols for c in comps] == [(0, 1364), (1364, 3412), (3412, 4112)]
        assert [c.n for c in comps] == [1364, 2048, 700]
        assert [c.world_offset for c in comps] == [31 * rank, 128 * rank, 14 * rank]
    comps = ppo_stage1.mix_components(parse_mix('circle:3,stage2:2'), None, 2)
    assert [(c.cols, c.world_offset) for c in comps] == [((0, 150), 6), ((150, 238), 4)]


def test_shards_tile_the_global_worlds():
    """Over R ranks, each component's world ranges [offset, offset + W_k) tile 0 .. R W_k - 1 exactly once."""
    from rl_collision_avoidance_b200.mix import parse_mix, plan
    mix = parse_mix('random:5,stage2:3,circle:2')
    robots = {'random': 8, 'stage2': 44, 'circle': 50}
    R = 3
    for k, (name, w) in enumerate(mix):
        ranges = sorted((plan(mix, robots, r)[k].world_offset, plan(mix, robots, r)[k].worlds) for r in range(R))
        covered = np.concatenate([np.arange(o, o + n) for o, n in ranges])
        assert np.array_equal(covered, np.arange(R * w)), name


def _views(ro, a, b):
    return dict(action=ro.scaled[a:b], stack=ro.stacks[:, a:b], gs=ro.gs[:, a:b], reward=ro.rewards[:, a:b],
                flags=ro.flags[:, a:b], eplog=ro.eplog[:, a:b])


def test_slices_of_512_beams_are_aligned():
    from rl_collision_avoidance_b200.mix import SLICE_ALIGN, check_aligned
    from rl_collision_avoidance_b200.trainer import Rollout
    ro = Rollout(4, 44 * 3 + 16 * 5 + 50, 512, 'cpu')
    for a, b in ((0, 132), (132, 212), (212, 262)):
        for name, v in _views(ro, a, b).items():
            check_aligned(name, v, SLICE_ALIGN[name])


def test_a_misaligned_slice_fails_loudly():
    """At 510 beams a FIFO frame is 2040 bytes, so every component's FIFO view fails, the first one included.  At 512
    beams a FIFO buffer that starts off the boundary fails on its start alone, as do gs and action buffers."""
    from rl_collision_avoidance_b200.mix import SLICE_ALIGN, check_aligned
    from rl_collision_avoidance_b200.trainer import Rollout
    ro = Rollout(4, 20, 510, 'cpu')
    for a, b in ((0, 20), (0, 7), (7, 20)):
        with pytest.raises(ValueError, match=r"stack is not 16-byte aligned \(start offset \d+ bytes, steps \[.*2040\]"):
            check_aligned('stack', ro.stacks[:, a:b], SLICE_ALIGN['stack'])
    frames = 5 * 20 * 3
    stack = torch.zeros(frames * 512 + 1)[1:].view(5, 20, 3, 512)   # starts 4 bytes past the boundary
    assert all(s * 4 % 16 == 0 for s in stack.stride()[:-1])         # every step is aligned: only the start is not
    with pytest.raises(ValueError, match=r'stack is not 16-byte aligned \(start offset 4 bytes'):
        check_aligned('stack', stack[:, 7:20], SLICE_ALIGN['stack'])
    check_aligned('stack', torch.zeros(frames * 512 + 4)[4:].view(5, 20, 3, 512)[:, 7:20], SLICE_ALIGN['stack'])
    base = torch.zeros(4 * 20 * 4 + 1)
    gs = base[1:].view(4, 20, 4)                      # starts 4 bytes past the boundary
    with pytest.raises(ValueError, match='gs is not 16-byte aligned'):
        check_aligned('gs', gs[:, 2:5], SLICE_ALIGN['gs'])
    a = torch.zeros(2 * 9 + 1)[1:].view(9, 2)
    with pytest.raises(ValueError, match='action is not 8-byte aligned'):
        check_aligned('action', a[3:6], SLICE_ALIGN['action'])
