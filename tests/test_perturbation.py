"""perturbation.Chain on recording fake links: the order of the links on both sides, the flags each gets, the gs the
policy reads in place and out of place, the settings and the refusals (DESIGN.md §9y).  The GPU tests pin the same
order bit for bit through the real links."""
import pytest

from rl_collision_avoidance_b200.perturbation import Chain


class _Link:
    """A fake link of `env` that appends (name, method, args) to `log` and returns a value naming itself"""

    def __init__(self, name, env, log, steer=True):
        self.name, self.env, self.log, self.steer = name, env, log, steer

    def _call(self, method, *args, **kw):
        self.log.append((self.name, method, args, kw))
        return '%s.%s' % (self.name, method)

    def action(self, cmd, *flags):
        return self._call('action', cmd, *flags)

    def scan(self, stack, flags):
        return self._call('scan', stack, flags)

    def observe(self, flags, gs=None, out=None):
        r = self._call('observe', flags, gs=gs, out=out)
        return out if out is not None else r

    def update(self, flags, reward, eplog, gs=None):
        out = self._call('update', flags, reward, eplog, gs=gs)
        return gs if gs is not None else out

    def settings(self):
        return {'link': self.name}


def _chain(env=None, steer=False, skip=()):
    env = object() if env is None else env
    log = []
    links = {k: None if k in skip else _Link(k, env, log, steer=steer)
             for k in ('noise', 'latency', 'dynamics', 'localization', 'planner')}
    return Chain(env, **links), log


def test_command_order_and_flags():
    chain, log = _chain()
    prev = object()
    assert chain.command('cmd', prev) == 'dynamics.action'
    assert [(n, m) for n, m, _, _ in log] == [('latency', 'action'), ('noise', 'action'), ('dynamics', 'action')]
    assert log[0][2] == ('cmd', prev)
    assert log[1][2] == ('latency.action',)
    assert log[2][2][0] == 'noise.action' and log[2][2][1] is log[0][2][1] is prev
    log.clear()
    chain.command('cmd', None)
    assert log[0][2] == ('cmd', None) and log[2][2] == ('noise.action', None)


def test_sense_order_start_and_returned_gs():
    chain, log = _chain(steer=True, skip=('localization',))
    assert chain.sense('stack') == 'planner.update'
    assert [(n, m) for n, m, _, _ in log] == [('latency', 'scan'), ('noise', 'scan'), ('planner', 'update')]
    assert all(args[-1] is None for n, m, args, _ in log if m == 'scan')
    assert log[2][2] == (None, None, None) and log[2][3] == {'gs': None}
    log.clear()
    flags = object()
    chain.sense('stack', flags)
    assert [args for _, _, args, _ in log] == [('stack', flags), ('stack', flags), (flags, None, None)]


def test_sense_localization_then_planner_without_steer():
    chain, log = _chain(steer=False)
    flags = object()
    assert chain.sense('stack', flags) == 'localization.observe'
    assert [(n, m) for n, m, _, _ in log] == [('latency', 'scan'), ('noise', 'scan'), ('localization', 'observe'),
                                              ('planner', 'update')]
    assert log[2][2] == (flags,) and log[2][3] == {'gs': None, 'out': None}
    assert log[3][3] == {'gs': None}                    # the planner reads env.gs, not localization's buffer


def test_sense_in_place():
    chain, log = _chain(steer=True, skip=('localization',))
    gs, flags, reward, eplog = object(), object(), object(), object()
    assert chain.sense('stack', flags, gs=gs, reward=reward, eplog=eplog) is gs
    assert log[2][2] == (flags, reward, eplog) and log[2][3]['gs'] is gs
    log.clear()
    chain.sense('stack', None, gs=gs)
    assert log[2][2] == (None, None, None) and log[2][3]['gs'] is gs


def test_sense_in_place_localization():
    chain, log = _chain(steer=False)
    gs, flags = object(), object()
    assert chain.sense('stack', flags, gs=gs) is gs
    assert log[2][2] == (flags,) and log[2][3]['gs'] is gs and log[2][3]['out'] is gs
    assert log[3][3]['gs'] is gs
    env = object()
    assert Chain(env).sense('stack') is None            # no link: the policy reads env.gs
    assert Chain(env).sense('stack', None, gs=gs) is gs


def test_settings():
    chain, _ = _chain(skip=('latency',))
    assert chain.settings() == {'noise': {'link': 'noise'}, 'dynamics': {'link': 'dynamics'},
                                'localization': {'link': 'localization'}}
    assert list(_chain(skip=('noise', 'dynamics'))[0].settings()) == ['latency', 'localization']


@pytest.mark.parametrize('name', ['noise', 'latency', 'dynamics', 'localization', 'planner'])
def test_refuses_a_link_of_another_env(name):
    env = object()
    with pytest.raises(ValueError, match='the %s belongs to another env' % name):
        Chain(env, **{name: _Link(name, object(), [])})


def test_refuses_a_steering_planner_with_localization():
    env = object()
    with pytest.raises(ValueError, match='localization error needs a planner on the believed pose'):
        Chain(env, localization=_Link('localization', env, []), planner=_Link('planner', env, [], steer=True))
    Chain(env, localization=_Link('localization', env, []), planner=_Link('planner', env, [], steer=False))
