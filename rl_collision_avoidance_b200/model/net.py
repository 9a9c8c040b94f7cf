"""CNNPolicy over the hand-written CUDA learner (mirror of /root/reference/model/net.py:16-80).

Same constructor, same `forward` / `evaluate_actions` return tuples and the same 23 state_dict keys
and shapes (SURVEY.md App. C), so the reference's `policy/*.pth` load unchanged.  The parameters are
views into ONE flat fp32 buffer (tensor starts padded to 32 floats): the optimizer is one fused
kernel and a data-parallel run all-reduces one buffer.  All math runs in librlca.so
(csrc/rlca_policy.cu); torch only owns the memory.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict

import torch

from .. import _lib

# state_dict order of the reference module (model/net.py:19-34)
TENSORS = [
    ('logstd', (2,)),
    ('act_fea_cv1.weight', (32, 3, 5)), ('act_fea_cv1.bias', (32,)),
    ('act_fea_cv2.weight', (32, 32, 3)), ('act_fea_cv2.bias', (32,)),
    ('act_fc1.weight', (256, 4096)), ('act_fc1.bias', (256,)),
    ('act_fc2.weight', (128, 260)), ('act_fc2.bias', (128,)),
    ('actor1.weight', (1, 128)), ('actor1.bias', (1,)),
    ('actor2.weight', (1, 128)), ('actor2.bias', (1,)),
    ('crt_fea_cv1.weight', (32, 3, 5)), ('crt_fea_cv1.bias', (32,)),
    ('crt_fea_cv2.weight', (32, 32, 3)), ('crt_fea_cv2.bias', (32,)),
    ('crt_fc1.weight', (256, 4096)), ('crt_fc1.bias', (256,)),
    ('crt_fc2.weight', (128, 260)), ('crt_fc2.bias', (128,)),
    ('critic.weight', (1, 128)), ('critic.bias', (1,)),
]
NPARAMS = 2172101


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class ParamList(list):
    """`policy.parameters()`: the named views, plus a back-reference for the fused optimizer."""
    policy = None


class CNNPolicy:
    def __init__(self, frames=3, action_space=2, device='cuda:0', seed=None, max_batch=1024):
        if frames != 3 or action_space != 2:
            raise ValueError('the CUDA learner is specialised for frames=3, action_space=2 (ppo_stage1.py:24,34)')
        if not torch.cuda.is_available():
            raise _lib.RlcaError('CNNPolicy needs a CUDA device: the learner has no CPU path')
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.offsets = [int(self.lib.rlca_policy_param_offset(i)) for i in range(len(TENSORS) + 1)]
        self.flat_size = self.offsets[-1]
        self.flat = torch.zeros(self.flat_size, device=self.device)
        self.grad = torch.zeros(self.flat_size, device=self.device)
        self.views = OrderedDict()
        self.grad_views = OrderedDict()
        for i, (name, shape) in enumerate(TENSORS):
            n = math.prod(shape)
            assert n == int(self.lib.rlca_policy_param_size(i))
            self.views[name] = self.flat[self.offsets[i]:self.offsets[i] + n].view(shape)
            self.grad_views[name] = self.grad[self.offsets[i]:self.offsets[i] + n].view(shape)
        self._ws = None
        self._ws_batch = 0
        self.max_batch = max_batch
        self.sample_seed = 0 if seed is None else int(seed)
        self.sample_counter = 0
        self.tensor_cores = True
        self.reset_parameters(seed)

    # ------------------------------------------------------------------ parameters
    def reset_parameters(self, seed=None):
        """PyTorch's default Conv1d/Linear init (kaiming_uniform(a=sqrt(5)) => U(+-1/sqrt(fan_in)) for
        weight and bias), logstd = 0 (model/net.py:19)."""
        gen = torch.Generator(device='cpu')
        gen.manual_seed(0 if seed is None else int(seed))
        for name, shape in TENSORS:
            v = self.views[name]
            if name == 'logstd':
                v.zero_()
                continue
            layer = name.rsplit('.', 1)[0]
            wshape = dict(TENSORS)[layer + '.weight']
            fan_in = math.prod(wshape[1:])
            bound = 1.0 / math.sqrt(fan_in)
            v.copy_(((torch.rand(shape, generator=gen) * 2 - 1) * bound).to(self.device))
        self.weights_changed()

    def rebind_storage(self, flat, grad):
        """Move the flat parameter / gradient buffers into caller-provided storage (e.g. a symmetric-memory allocation
        that the other ranks can address); contents are copied, the named views are rebuilt."""
        flat.copy_(self.flat)
        grad.copy_(self.grad)
        self.flat, self.grad = flat, grad
        for i, (name, shape) in enumerate(TENSORS):
            n = math.prod(shape)
            self.views[name] = self.flat[self.offsets[i]:self.offsets[i] + n].view(shape)
            self.grad_views[name] = self.grad[self.offsets[i]:self.offsets[i] + n].view(shape)
        self.weights_changed()

    def weights_changed(self):
        """Call after writing to the parameter buffer outside Adam.step / load_state_dict."""
        if getattr(self, '_ws', None) is not None:
            _lib.check(self.lib.rlca_policy_weights_changed(self._ws))

    def parameters(self):
        pl = ParamList(self.views.values())
        pl.policy = self
        return pl

    def named_parameters(self):
        return list(self.views.items())

    def state_dict(self):
        return OrderedDict((k, v.detach().clone()) for k, v in self.views.items())

    def load_state_dict(self, sd, strict=True):
        missing = [k for k in self.views if k not in sd]
        extra = [k for k in sd if k not in self.views]
        if strict and (missing or extra):
            raise KeyError(f'state_dict mismatch: missing {missing}, unexpected {extra}')
        for k, v in self.views.items():
            if k in sd:
                v.copy_(sd[k].to(device=self.device, dtype=torch.float32).view(v.shape))
        self.weights_changed()
        return self

    def cuda(self):
        return self

    def zero_grad(self):
        self.grad.zero_()

    # ------------------------------------------------------------------ workspace
    @property
    def launch_count(self):
        """Kernel launches issued through this policy's workspace (rlca_policy_launch_count)."""
        return int(self.lib.rlca_policy_launch_count(self._ws)) if self._ws is not None else 0

    def _workspace(self, nb):
        if self._ws is None or nb > self._ws_batch:
            if self._ws is not None:
                self.lib.rlca_policy_destroy(self._ws)
            cap = max(nb, self.max_batch)
            h = C.c_void_p()
            torch.cuda.set_device(self.device)
            _lib.check(self.lib.rlca_policy_create(cap, C.byref(h)))
            self._ws, self._ws_batch = h, cap
            _lib.check(self.lib.rlca_policy_set_tensor_cores(self._ws, int(self.tensor_cores)))
        return self._ws

    def set_tensor_cores(self, enable=True):
        """Conv tower + fc1 GEMMs on wgmma with 3xTF32 compensation (True, default), fc1 GEMMs only (2),
        or everything on the fp32 CUDA-core kernels (False)."""
        self.tensor_cores = 2 if enable == 2 and enable is not True else bool(enable)
        if self._ws is not None:
            _lib.check(self.lib.rlca_policy_set_tensor_cores(self._ws, int(self.tensor_cores)))

    def features(self, tower, nb):
        """relu(conv2) features (nb, 4096) of the last forward, tower 0 actor / 1 critic (inspection hook)."""
        out = torch.empty(nb, 4096, device=self.device)
        _lib.check(self.lib.rlca_policy_features(self._ws, tower, nb, _ptr(out), self._stream()))
        return out

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def __del__(self):
        try:
            if self._ws is not None:
                self.lib.rlca_policy_destroy(self._ws)
        except Exception:
            pass

    @staticmethod
    def _pack_gs(goal, speed):
        return torch.cat((goal, speed), dim=-1).contiguous()

    # ------------------------------------------------------------------ reference surface
    def forward_values(self, x, gs, v_out=None, mean_out=None):
        """value (nb,), mean (nb,2) without sampling; keeps activations for backward."""
        nb = x.shape[0]
        x = x.contiguous()
        v = v_out if v_out is not None else torch.empty(nb, device=self.device)
        mean = mean_out if mean_out is not None else torch.empty(nb, 2, device=self.device)
        _lib.check(self.lib.rlca_policy_forward(self._workspace(nb), _ptr(self.flat), _ptr(x), _ptr(gs), nb,
                                                _ptr(v), _ptr(mean), self._stream()))
        return v, mean

    def forward(self, x, goal, speed, gs=None, out=None):
        """returns value estimation, action, log_action_prob, mean  (model/net.py:37-70).
        `out` may hold preallocated 'value' (nb,), 'action' (nb,2), 'logprob' (nb,), 'scaled' (nb,2) tensors
        (rollout slices); 'scaled' receives the clipped action of model/ppo.py:75."""
        out = out or {}
        gs = gs if gs is not None else self._pack_gs(goal, speed)
        v, mean = self.forward_values(x, gs, out.get('value'), out.get('mean'))
        nb = x.shape[0]
        action = out['action'] if 'action' in out else torch.empty(nb, 2, device=self.device)
        logprob = out['logprob'] if 'logprob' in out else torch.empty(nb, device=self.device)
        self.sample_counter += 1
        _lib.check(self.lib.rlca_policy_sample(_ptr(self.flat), _ptr(mean), nb, self.sample_seed, self.sample_counter,
                                               0, _ptr(action), _ptr(logprob), _ptr(out.get('scaled')), self._stream()))
        return v.view(nb, 1), action, logprob.view(nb, 1), mean

    __call__ = forward

    def evaluate_actions(self, x, goal, speed, action, gs=None):
        """(v, logprob, dist_entropy) for given actions (model/net.py:72-80)"""
        gs = gs if gs is not None else self._pack_gs(goal, speed)
        v, mean = self.forward_values(x, gs)
        nb = x.shape[0]
        action = action.contiguous()
        logprob = torch.empty(nb, device=self.device)
        _lib.check(self.lib.rlca_policy_sample(_ptr(self.flat), _ptr(mean), nb, 0, 0, 2, _ptr(action), _ptr(logprob),
                                               C.c_void_p(0), self._stream()))
        logstd = self.views['logstd']
        dist_entropy = (0.5 + 0.5 * math.log(2 * math.pi) + logstd).sum()
        return v.view(nb, 1), logprob.view(nb, 1), dist_entropy


class Adam:
    """torch.optim.Adam(policy.parameters(), lr) mirror (ppo_stage1.py:179): one fused kernel over the flat
    parameter buffer.  `grad_scale` lets a data-parallel caller fold the 1/world_size of the gradient
    average into the update."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        policy = getattr(params, 'policy', None) or params
        if not isinstance(policy, CNNPolicy):
            raise TypeError('pass policy.parameters() (or the CNNPolicy) to Adam')
        self.policy = policy
        self.lr, self.betas, self.eps = lr, betas, eps
        self.exp_avg = torch.zeros_like(policy.flat)
        self.exp_avg_sq = torch.zeros_like(policy.flat)
        self.step_count = 0
        self.peer = None          # data-parallel run: the fused all-reduce + Adam over peer memory (parallel.PeerAdam)

    def zero_grad(self):
        self.policy.grad.zero_()

    def step(self, grad_scale=1.0):
        p = self.policy
        self.step_count += 1
        if self.peer is not None:           # gradient sum over the ranks, Adam and the broadcast of the result: one kernel
            self.peer.step(self, grad_scale)
            p.weights_changed()
            return
        # one kernel: Adam over the flat buffer + the tf32 hi / lo split (and transposes) of the fc1 weights that the
        # tensor-core GEMMs of the next forward / backward read; it marks the workspace's other weight images stale
        _lib.check(p.lib.rlca_policy_adam_step(p._workspace(1), _ptr(p.flat), _ptr(p.grad), _ptr(self.exp_avg),
                                               _ptr(self.exp_avg_sq), self.lr, self.betas[0], self.betas[1], self.eps,
                                               self.step_count, grad_scale, p._stream()))

    def state_dict(self):
        if self.peer is not None:           # sharded moments: read the other ranks' shards through the peer mappings
            m, v = self.peer.gather_moments()
        else:
            m, v = self.exp_avg.clone(), self.exp_avg_sq.clone()
        return {'exp_avg': m, 'exp_avg_sq': v, 'step': self.step_count, 'lr': self.lr, 'betas': self.betas, 'eps': self.eps}

    def load_state_dict(self, sd):
        self.exp_avg.copy_(sd['exp_avg'])
        self.exp_avg_sq.copy_(sd['exp_avg_sq'])
        self.step_count = int(sd['step'])
