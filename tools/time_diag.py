"""What the PPO update diagnostics cost (DESIGN.md §9n): the 1024-row minibatch step - forward, loss, backward, Adam, as
bench.py's learner section runs it - with the diagnostics off and on, alternated in one process and timed with CUDA
events after a warm-up; then, in a run of its own under torch.profiler, the device time of the three diagnostics
kernels inside that step; and the enqueue rate of the two entries called back to back from Python.  Prints the card
and power limit first.  There is no measurement without a GPU."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from rl_collision_avoidance_b200 import _lib
from rl_collision_avoidance_b200.model.diagnostics import PPODiagnostics
from rl_collision_avoidance_b200.model.net import Adam, CNNPolicy, _ptr

NB, ROUNDS, STEPS, WARM, PROFILED, ALONE = 1024, 8, 200, 20, 50, 2000


def timed(fn, n):
    """us per call of fn over n calls (CUDA events on the current stream)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


def main():
    if not torch.cuda.is_available():
        raise SystemExit('time_diag.py needs a CUDA device')
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        power = 'unknown'
    print('card: %s, power limit: %s' % (torch.cuda.get_device_name(0), power))
    dev = 'cuda'
    pol = CNNPolicy(max_batch=NB, seed=0)
    opt = Adam(pol.parameters(), lr=5e-5)
    diag = PPODiagnostics(pol, 1, [[0, -1], [1, 1]])
    lib = pol.lib
    obs = torch.rand(NB, 1536, device=dev) - 0.5
    gs = torch.rand(NB, 4, device=dev)
    v, mean = torch.empty(NB, device=dev), torch.empty(NB, 2, device=dev)
    act, lp = torch.rand(NB, 2, device=dev), torch.rand(NB, device=dev) - 1
    adv, tgt, losses = torch.randn(NB, device=dev), torch.randn(NB, device=dev), torch.zeros(3, device=dev)
    ws, st = pol._workspace(NB), pol._stream()

    def step(on):
        _lib.check(lib.rlca_policy_forward(ws, _ptr(pol.flat), _ptr(obs), _ptr(gs), NB, _ptr(v), _ptr(mean), st))
        _lib.check(lib.rlca_ppo_loss_fwd_bwd(ws, _ptr(pol.flat), _ptr(v), _ptr(mean), _ptr(act), _ptr(lp), _ptr(adv),
                                             _ptr(tgt), NB, 0.1, 5e-4, 20.0, _ptr(losses), st))
        if on:
            diag.accumulate(0, v, mean, act, lp, adv, tgt, NB, 0.1)
        _lib.check(lib.rlca_policy_backward(ws, _ptr(pol.flat), _ptr(obs), _ptr(gs), NB, _ptr(pol.grad), st))
        if on:
            diag.grads(0)
        opt.step()

    for on in (False, True):
        for _ in range(WARM):
            step(on)
    torch.cuda.synchronize()
    off, on = [], []
    for _ in range(ROUNDS):
        off.append(timed(lambda: step(False), STEPS))
        on.append(timed(lambda: step(True), STEPS))
    for name, t in (('off', off), ('on', on)):
        print('minibatch step of %d rows, diagnostics %s: %.1f us (mean of %d windows of %d steps; min %.1f, max %.1f)'
              % (NB, name, np.mean(t), ROUNDS, STEPS, min(t), max(t)))
    d = np.array(on) - np.array(off)
    print('difference on - off: %.1f us (%.2f %% of the step; per window min %.1f, max %.1f)'
          % (d.mean(), 100 * d.mean() / np.mean(off), d.min(), d.max()))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(PROFILED):
            step(True)
        torch.cuda.synchronize()
    nbytes = 4 * sum(p.numel() for p in pol.parameters())
    for e in prof.key_averages():
        if any(k in e.key for k in ('ppo_diag_kernel', 'grad_sumsq_kernel', 'grad_sumsq_final_kernel')):
            us = e.device_time_total / e.count
            note = ', %.2f MB read, %.0f GB/s' % (nbytes / 1e6, nbytes / us / 1e3) if 'grad_sumsq_kernel' in e.key else ''
            print('device time inside the step (torch.profiler, %d launches): %s %.2f us%s'
                  % (e.count, e.key.split('(')[0], us, note))
    acc_us = timed(lambda: diag.accumulate(0, v, mean, act, lp, adv, tgt, NB, 0.1), ALONE)
    grad_us = timed(lambda: diag.grads(0), ALONE)
    print('called back to back from Python: rlca_ppo_diag_accumulate %.1f us, '
          'rlca_grad_sumsq %.1f us per call (mean of %d calls each)' % (acc_us, grad_us, ALONE))


if __name__ == '__main__':
    main()
