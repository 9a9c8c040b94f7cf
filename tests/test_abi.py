"""The C-ABI library loads without a GPU and exports every symbol include/rlca.h declares."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, 'include', 'rlca.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(rlca_[a-z0-9_]+)\s*\(', src)))


def test_library_exports_every_declared_symbol(built):
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    names = header_functions()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/rlca.h but not exported by librlca.so'
        assert n in _lib.SYMBOLS, f'{n} has no ctypes signature in _lib.SYMBOLS'
    assert sorted(_lib.SYMBOLS) == names
    assert b'sm_90a' in lib.rlca_version()


def test_config_struct_layout_matches_c(built):
    from rl_collision_avoidance_b200 import _lib
    lib = _lib.load()
    assert lib.rlca_sizeof_env_config() == C.sizeof(_lib.EnvConfig)


def test_no_gpu_means_loud_failure(built):
    import torch
    from rl_collision_avoidance_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    lib = _lib.load()
    from rl_collision_avoidance_b200.scenarios import fill_config, make_scenario
    cfg = fill_config(_lib.EnvConfig(), make_scenario('stage1'), num_worlds=1, beams=512)
    h = C.c_void_p()
    rc = lib.rlca_env_create(C.byref(cfg), C.byref(h))
    assert rc == 4 and b'no CPU fallback' in lib.rlca_last_error()
    from rl_collision_avoidance_b200.stage_world import StageWorld
    with pytest.raises(_lib.RlcaError):
        StageWorld(512, scenario='stage1')


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, 'rl_collision_avoidance_b200')
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh', '.h')):
                txt = open(os.path.join(dirpath, f)).read()
                assert 'import oracle' not in txt and 'from oracle' not in txt and 'sim_oracle' not in txt.replace(
                    'oracle/sim_oracle.c', ''), f'{f} references the oracle'
