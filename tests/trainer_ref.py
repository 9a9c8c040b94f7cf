"""Numpy / float64 restatement of the reference's training loop (ppo_stage1.py:39-131, ppo_stage2.py:39-138,
model/ppo.py:111-259, model/utils.py:65-78), written from those rules, not from rl_collision_avoidance_b200/trainer.py.

The network, the log-probability and the PPO losses are learner_ref.ref_forward / ref_logprob / ref_losses; this
module holds what the loop adds around them:

* the per-robot scan deque: [obs] * 3 at an episode start (ppo_stage1.py:59-60), popleft / append after each tick
  (:87-89), with the local goal and speed read after the tick (:90-91);
* stage 2's liveflag (ppo_stage2.py:55,72-84): a robot whose episode ended idles until its whole group has ended; its
  buffer row keeps the last reward it got (`r` is not reassigned) and terminal stays true;
* the GAE recurrence (model/ppo.py:122-139);
* get_filter_index (model/utils.py:65-78), whose run counter is not reset between columns;
* the advantage normalisation over all H x N rows with numpy's population std, before np.delete (model/ppo.py:148 and
  :202 before :212-218);
* the minibatch schedules: BatchSampler(SubsetRandomSampler(range(n)), batch_size, drop_last) with drop_last False
  in stage 1 (:159-160, a ragged last minibatch) and True in stage 2 (:222-223, the tail dropped);
* Adam with torch.optim.Adam's rule (ppo_stage1.py:179): bias corrections, eps added to sqrt(v / bc2) (after the bias
  correction), the step lr / bc1 * m / denom."""
from collections import deque

import numpy as np


# ------------------------------------------------------------------------------------------------ the scan deque
def scan_deque(obs):
    """the observation stack of an episode start: deque([obs, obs, obs]) (ppo_stage1.py:59-60)"""
    return deque([obs, obs, obs])


def push(stack, obs):
    """the tick's new scan enters the stack: popleft, append (ppo_stage1.py:87-89)"""
    stack.popleft()
    stack.append(obs)
    return stack


class Stacks:
    """One scan deque per robot.  tick(obs, restart): a robot flagged in `restart` starts a new episode from the scan
    of its new pose (the next pass of ppo_stage1.py:51-60); every other robot pushes its new scan."""

    def __init__(self, obs):
        self.q = [scan_deque(o.copy()) for o in obs]

    def tick(self, obs, restart):
        for i, o in enumerate(obs):
            if restart[i]:
                self.q[i] = scan_deque(o.copy())
            else:
                push(self.q[i], o.copy())

    def array(self):
        """(N, 3, beams): the oldest frame first, as the deque is handed to the policy"""
        return np.stack([np.stack(list(q)) for q in self.q])

    def load(self, arr):
        """replace every deque's frames by the rows of `arr` (a perturbed copy of array())"""
        self.q = [deque([a[0].copy(), a[1].copy(), a[2].copy()]) for a in arr]


# ------------------------------------------------------------------------------------------------ stage 2's liveflag
def liveflag_rows(live_ticks, ticks):
    """The (r, terminal) of one stage-2 robot's buffer rows over `ticks` ticks of its group's episode.  `live_ticks`
    holds the (r, terminal) that get_reward_and_terminate returned on each tick while liveflag was true, the last one
    terminal.  Once terminal, the robot idles: control_vel and get_reward_and_terminate are skipped (ppo_stage2.py:72-
    79), so `r` keeps its last value and `terminal` stays true (:83-84).  The GPU replay of trainer.run takes the rows
    from the CPU oracle, which implements this rule and is held to the reference elsewhere; it checks the rule on them
    (an idle row repeats the robot's last reward, done 1, result 0)."""
    rows = []
    live, r, terminal = True, 0.0, False
    it = iter(live_ticks)
    for _ in range(ticks):
        if live:
            r, terminal = next(it)
        if terminal:
            live = False
        rows.append((r, terminal))
    return rows


# ------------------------------------------------------------------------------------------------ the update's data
def gae(rewards, values, last_value, dones, gamma, lam):
    """model/ppo.py:122-139 in float64: (targets, advantages), both (T, N)"""
    r, v, d = (np.asarray(a, np.float64) for a in (rewards, values, dones))
    T, N = r.shape
    vals = np.concatenate([v, np.asarray(last_value, np.float64).reshape(1, N)])
    targets = np.zeros((T, N))
    g = np.zeros(N)
    for t in range(T - 1, -1, -1):
        delta = r[t] + gamma * vals[t + 1] * (1 - d[t]) - vals[t]
        g = delta + gamma * lam * (1 - d[t]) * g
        targets[t] = g + vals[t]
    return targets, targets - vals[:-1]


def filter_index(d_list):
    """model/utils.py:65-78: flat indices num_env * j + i of the second and later done of a run, the columns walked one
    after the other with ONE counter, so a run of dones at the end of column i continues at the top of column i + 1"""
    d = np.asarray(d_list)
    step, num_env = d.shape
    out, flag = [], 0
    for i in range(num_env):
        for j in range(step):
            flag = flag + 1 if d[j, i] else 0
            if flag >= 2:
                out.append(num_env * j + i)
    return out


def normalise(advs):
    """(advs - advs.mean()) / advs.std() over every row of the rollout, numpy's population std (model/ppo.py:148,202)"""
    a = np.asarray(advs, np.float64)
    return (a - a.mean()) / a.std()


def kept_rows(n_all, filter_idx):
    """the row numbers np.delete(x, filter_index, 0) keeps (model/ppo.py:212-218), in order"""
    return np.delete(np.arange(n_all), np.asarray(filter_idx, np.int64))


def minibatches(perm, batch_size, drop_last):
    """BatchSampler over a SubsetRandomSampler whose order is `perm`: consecutive chunks of batch_size; the last, short
    chunk is kept (stage 1, model/ppo.py:159-160) or dropped (stage 2, :222-223)"""
    perm = np.asarray(perm)
    out = [perm[k:k + batch_size] for k in range(0, len(perm), batch_size)]
    if drop_last and out and len(out[-1]) < batch_size:
        out.pop()
    return out


# ------------------------------------------------------------------------------------------------ Adam
def adam_step(p, g, m, v, step, lr, betas=(0.9, 0.999), eps=1e-8):
    """One torch.optim.Adam step in float64 (step counts from 1): returns the new (p, m, v).
    m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2, denom = sqrt(v) / sqrt(1 - b2^step) + eps,
    p -= lr / (1 - b1^step) * m / denom."""
    b1, b2 = (float(b) for b in betas)
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    m = b1 * m + (1.0 - b1) * g
    v = b2 * v + (1.0 - b2) * g * g
    denom = np.sqrt(v) / np.sqrt(1.0 - b2 ** step) + eps
    return p - lr / (1.0 - b1 ** step) * (m / denom), m, v
