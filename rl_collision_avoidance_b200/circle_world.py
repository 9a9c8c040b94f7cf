"""Circle-swap env client (mirror of /root/reference/circle_world.py): 50 robots on a 25 m circle,
antipodal goals, |w| > 0.7 penalty, timeout 10000.  `num_env=K` / `radius=r` place K robots on a circle of r metres
instead (scenarios.circle_layout); the defaults keep the reference's 50-row table."""
from .scenarios import make_scenario
from .stage_world import StageWorld as _Base


class StageWorld(_Base):
    def __init__(self, beam_num, index=0, num_env=50, radius=None, **kw):
        if 'scenario' not in kw:
            kw['scenario'] = make_scenario('circle', kw.pop('map', None), num_env, radius)
        super().__init__(beam_num, index, num_env, **kw)
