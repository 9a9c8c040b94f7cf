"""The SL-policy without a device: the driver's argument checks and the register / spill budget of the new kernels."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('argv, message', [
    (['--samples', '0'], '--samples must be >= 1'),
    (['--num-worlds', '0'], '--num-worlds must be >= 1'),
    (['--record-every', '0'], '--record-every must be >= 1'),
    (['--epochs', '0'], '--epochs must be >= 1'),
    (['--batch-size', '0'], '--batch-size must be >= 1'),
    (['--lr', '0'], '--lr must be finite and > 0'),
    (['--lr', 'nan'], '--lr must be finite and > 0'),
    (['--holdout', '1'], '--holdout must be in [0, 1)'),
    (['--holdout', '-0.1'], '--holdout must be in [0, 1)'),
    (['--scenario', 'stage3'], 'invalid choice'),
    (['--orca-gain', '2'], '--orca-gain applies to --baseline orca only'),
    (['--no-orca-map', '--orca-obstacle-horizon', '1'], '--orca-obstacle-horizon applies with --orca-map only'),
])
def test_sl_train_rejects_bad_arguments(tmp_path, capsys, argv, message):
    import sl_train
    with pytest.raises(SystemExit) as e:
        sl_train.parse(argv + ['--out', str(tmp_path / 'sl.pth')])
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_sl_train_rejects_missing_out_directory(tmp_path, capsys):
    import sl_train
    with pytest.raises(SystemExit):
        sl_train.parse(['--out', str(tmp_path / 'missing' / 'sl.pth')])
    assert 'does not exist' in capsys.readouterr().err


def test_sl_train_defaults():
    import sl_train
    a = sl_train.parse(['--out', 'sl.pth'])
    assert a.scenario == ['stage1', 'stage2'] and a.samples * len(a.scenario) == 800000
    assert a.baseline == 'nh-orca' and a.orca_map and a.batch_size == 1024
    assert sl_train.parse(['--out', 'sl.pth', '--scenario', 'circle', '--scenario', 'stage1']).scenario == \
        ['circle', 'stage1']
    assert not sl_train.parse(['--out', 'sl.pth', '--no-orca-map']).orca_map


@pytest.mark.parametrize('obj, kernel', [('rlca_demo.o', 'demo_append_kernel'), ('rlca_policy.o', 'bc_loss_kernel')])
def test_new_kernels_do_not_spill(built, obj, kernel):
    import __graft_entry__ as g
    cuobjdump = os.path.join(os.path.dirname(g.NVCC), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-res-usage', os.path.join(g.PKG, 'build', obj)], check=True,
                         capture_output=True, text=True).stdout
    m = re.search(r'Function \w*%s\w*:\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)' % kernel, out)
    assert m, out
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, m.group(0)
    assert int(m.group(1)) <= 64, m.group(0)
