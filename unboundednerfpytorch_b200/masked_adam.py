"""MaskedAdam with the reference's constructor / step surface (FourierGrid/masked_adam.py:21-75).

* per-voxel learning rate (``set_pervoxel_lr``), masked update (skip elements whose grad is exactly 0).
* ``step()`` dispatches per parameter to the adam_upd / masked_adam_upd / adam_upd_with_perlr kernels
  (adam_upd_kernel.cu:9-58) exactly like masked_adam.py:62-75.
"""
import torch

from . import ops


class MaskedAdam(torch.optim.Optimizer):

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.99), eps=1e-8):
        if not 0.0 <= lr:
            raise ValueError('Invalid learning rate: {}'.format(lr))
        if not 0.0 <= eps:
            raise ValueError('Invalid epsilon value: {}'.format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError('Invalid beta parameter at index 0: {}'.format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError('Invalid beta parameter at index 1: {}'.format(betas[1]))
        self.per_lr = None
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))

    def set_pervoxel_lr(self, count):
        assert self.param_groups[0]['params'][0].shape == count.shape
        self.per_lr = count.float() / count.max()

    def _begin(self, param):
        """Per-parameter bookkeeping of one optimizer step (state allocation + step counter, masked_adam.py:52-58)."""
        state = self.state[param]
        if len(state) == 0:
            state['step'] = 0
            state['exp_avg'] = torch.zeros_like(param, memory_format=torch.preserve_format)
            state['exp_avg_sq'] = torch.zeros_like(param, memory_format=torch.preserve_format)
        state['step'] += 1
        return state

    def _apply(self, group, param, state, sl=None):
        """Run the update kernel on `param` (or on its leading-dim slice `sl`, used by the slab-pipelined
        multi-GPU tail in dist.reduce_tv_step) -- same dispatch as masked_adam.py:62-75."""
        lr, (beta1, beta2), eps = group['lr'], group['betas'], group['eps']
        grad = param.grad
        if grad.stride() != param.stride():
            grad = torch.empty_like(param, memory_format=torch.preserve_format).copy_(grad)
        per_lr = None
        if self.per_lr is not None and param.shape == self.per_lr.shape:
            per_lr = self.per_lr
            if per_lr.stride() != param.stride():
                per_lr = torch.empty_like(param, memory_format=torch.preserve_format).copy_(per_lr)
                self.per_lr = per_lr
        cut = (lambda t: t) if sl is None else (lambda t: t[sl])
        p, g, m, v = cut(param), cut(grad), cut(state['exp_avg']), cut(state['exp_avg_sq'])
        if per_lr is not None:
            ops.adam_upd_with_perlr(p, g, m, v, cut(per_lr), state['step'], beta1, beta2, lr, eps)
        elif group['skip_zero_grad']:                     # KeyError when absent, like masked_adam.py:49
            ops.masked_adam_upd(p, g, m, v, state['step'], beta1, beta2, lr, eps)
        else:
            ops.adam_upd(p, g, m, v, state['step'], beta1, beta2, lr, eps)

    @torch.no_grad()
    def step_fused_tv(self, tv=None, write_grad=True):
        """``total_variation_add_grad`` on the grids listed in ``tv`` ({param: (wx, wy, wz, dense_mode)}) + ``step()`` with the
        two full-grid sweeps merged into one for channels-last grids (ops.tv_adam_pingpong): the updated parameters are
        written into a second buffer and the parameter's storage is swapped with it (state key 'pingpong', allocated on
        first use: +1 grid of memory).  Same result as the two calls, bit for bit."""
        tv = tv or {}
        for group in self.param_groups:
            group['skip_zero_grad']
            for param in group['params']:
                if param.grad is None:
                    continue
                state = self._begin(param)
                fused = (param in tv and self.per_lr is None and ops.tv_adam_pingpong_supported(param)
                         and param.grad.stride() == param.stride())
                if not fused:
                    if param in tv:
                        ops.total_variation_add_grad(param, param.grad, *tv[param])
                    self._apply(group, param, state)
                    continue
                if 'pingpong' not in state:
                    state['pingpong'] = torch.empty_like(param, memory_format=torch.preserve_format)
                wx, wy, wz, dense = tv[param]
                (beta1, beta2) = group['betas']
                ops.tv_adam_pingpong(param.data, state['pingpong'], param.grad, state['exp_avg'], state['exp_avg_sq'], wx, wy, wz,
                                     dense, state['step'], beta1, beta2, group['lr'], group['eps'],
                                     skip_zero_grad=group['skip_zero_grad'], write_grad=write_grad)
                old = param.data
                param.data = state['pingpong']
                state['pingpong'] = old

    def zero_grad(self, set_to_none=True):
        """torch.optim.Optimizer.zero_grad; a parameter that owns a persistent gradient buffer (dist.PeerTail) has the BUFFER
        zeroed when it still holds an unconsumed gradient, and .grad detached from it."""
        for group in self.param_groups:
            for param in group['params']:
                buf = getattr(param, '_ubn_grad_buffer', None)
                if buf is not None and param.grad is not None:
                    buf.zero_()
                    param.grad = None
        super().zero_grad(set_to_none=set_to_none)

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            group['skip_zero_grad']                       # KeyError when absent, like masked_adam.py:49
            for param in group['params']:
                if param.grad is None:
                    continue
                self._apply(group, param, self._begin(param))


def create_optimizer_or_freeze_model(model, cfg_train, global_step, verbose=False):
    """Optimizer factory with the reference's config keys (FourierGrid/utils.py:26-56): every ``lrate_<name>``
    key names a sub-module / parameter of ``model``; lr decays by 0.1 every ``lrate_decay``*1000 steps;
    ``skip_zero_grad_fields`` selects the masked update.  ``verbose`` is accepted for the reference's signature
    (run_train.py:54 passes it) and logs nothing."""
    get = (lambda k, d=None: cfg_train.get(k, d)) if hasattr(cfg_train, 'get') else (lambda k, d=None: getattr(cfg_train, k, d))
    keys = cfg_train.keys() if hasattr(cfg_train, 'keys') else vars(cfg_train).keys()
    decay_steps = get('lrate_decay') * 1000
    decay_factor = 0.1 ** (global_step / decay_steps)
    skip = get('skip_zero_grad_fields', []) or []
    groups = []
    for k in keys:
        if not k.startswith('lrate_') or k == 'lrate_decay':
            continue
        name = k[len('lrate_'):]
        if not hasattr(model, name):
            continue
        param = getattr(model, name)
        if param is None:
            continue
        lr = get(k) * decay_factor
        if lr > 0:
            if isinstance(param, torch.nn.Module):
                param = param.parameters()
            groups.append({'params': param, 'lr': lr, 'skip_zero_grad': (name in skip)})
        else:
            if isinstance(param, torch.nn.Module):
                for p in param.parameters():
                    p.requires_grad = False
            else:
                param.requires_grad = False
    return MaskedAdam(groups)
