"""The optimizer of the pre-training configs on the H100 (csrc/optim.cu): gradient-norm clip and AdamW over every
parameter in two launches, with mmcv's per-parameter learning-rate groups.

Every ViDAR config asks for
    optimizer = dict(type='AdamW', lr=2e-4, paramwise_cfg=dict(custom_keys={'img_backbone': dict(lr_mult=0.1)}),
                     weight_decay=0.01)
    optimizer_config = dict(grad_clip=dict(max_norm=35, norm_type=2))
which mmcv runs as one torch AdamW group per parameter tensor and a `clip_grad_norm_` before each step: thousands of
small launches and a host sync for the logged norm.  `AdamW(paramwise_groups(...), max_grad_norm=35)` computes the
same step (torch's single-tensor update after the clip, to fp32 rounding: the norm is summed in fp64) in one norm
launch and one update launch, on the current stream, with no host sync.  `pretrain.config_optimizer` builds it for
the harness; registered into mmcv as `VidarAdamW` (INTEGRATION.md)."""
import numpy as np
import torch

from . import _lib


def paramwise_groups(module, lr, weight_decay, custom_keys):
    """mmcv 1.4 `DefaultOptimizerConstructor.add_params` with `paramwise_cfg=dict(custom_keys=custom_keys)`: one group
    {'params': [p], 'lr', 'weight_decay'} per parameter in `named_parameters()` order.  The keys are tried longest
    first (ties in alphabetical order); the first that is a substring of the parameter's full name sets
    lr * lr_mult and weight_decay * decay_mult (both default 1).  A frozen parameter (requires_grad False) keeps the
    base values, as mmcv adds it before looking at the keys."""
    keys = sorted(sorted(custom_keys), key=len, reverse=True)
    groups = []
    for name, p in module.named_parameters():
        group = dict(params=[p], lr=lr, weight_decay=weight_decay)
        if p.requires_grad:
            for key in keys:
                if key in name:
                    group["lr"] = lr * custom_keys[key].get("lr_mult", 1.0)
                    group["weight_decay"] = weight_decay * custom_keys[key].get("decay_mult", 1.0)
                    break
        groups.append(group)
    return groups


class AdamW(torch.optim.Optimizer):
    """torch.optim.AdamW with the clip of mmcv's OptimizerHook folded in: `step()` clips every gradient to a total
    2-norm of `max_grad_norm` (None: no clip) and steps every parameter that has a gradient, in two launches (one
    without the clip; one more of each per 896 parameters or change of betas / eps).  The total norm is left in
    `self.grad_norm`, a 0-d fp32 device tensor, so a caller can log it without a sync.

    Takes a parameter list or groups (mmcv's one-tensor groups included); `group['lr']` and `group['weight_decay']`
    are read at every step, so LR schedulers and mmcv's LrUpdaterHook work, and so does `torch.amp.GradScaler`.  A
    parameter whose gradient is None is skipped as torch skips it.  Parameters and gradients must be fp32, dense,
    contiguous and on one CUDA device.  The state is torch's (`step`, `exp_avg`, `exp_avg_sq` per parameter; the
    moments are views into two flat buffers) and its state_dict loads into torch.optim.AdamW and back.  Parameter
    addresses are cached at the first step: replace a parameter's storage (`p.data = ...`) only before it, or rebuild
    the optimizer."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False,
                 max_grad_norm=None):
        if amsgrad:
            raise ValueError("vidar_b200.optim.AdamW does not implement amsgrad")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f"Invalid beta parameters: {betas}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if max_grad_norm is not None and not max_grad_norm > 0:
            raise ValueError(f"Invalid max_grad_norm: {max_grad_norm}")
        # torch.optim.AdamW's group keys, so that a state_dict of either optimizer loads into the other
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        self._flat = None
        super().__init__(params, defaults)
        self.max_grad_norm = max_grad_norm
        self.grad_norm = None

    def add_param_group(self, param_group):
        params = param_group["params"]
        params = [params] if isinstance(params, torch.Tensor) else list(params)
        device = next((p.device for g in self.param_groups for p in g["params"]), params[0].device if params else None)
        for p in params:
            if p.dtype != torch.float32 or not p.is_cuda:
                raise RuntimeError(f"vidar_b200.optim.AdamW takes fp32 CUDA parameters (got {p.dtype} on {p.device})")
            if not p.is_contiguous():
                raise RuntimeError("vidar_b200.optim.AdamW takes contiguous parameters")
            if p.device != device:
                raise RuntimeError(f"parameters on {device} and {p.device}: one device per optimizer")
        super().add_param_group(dict(param_group, params=params))
        self._flat = None                        # remade, with the state copied in, at the next step

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._flatten()

    def _params(self):
        return [p for g in self.param_groups for p in g["params"]]

    def _flatten(self):
        """(Re)make the cache: the parameters' addresses, numels and group of each, and the state as
        views into two flat fp32 buffers [sum numel] in parameter order and one CPU fp32 step vector, with whatever
        state the parameters already have copied in."""
        params = self._params()
        device = params[0].device if params else None
        n = len(params)
        numel = np.fromiter((p.numel() for p in params), np.int64, n)
        offset = np.zeros(n + 1, np.int64)
        np.cumsum(numel, out=offset[1:])
        total = int(offset[-1])
        exp_avg = torch.zeros(total, dtype=torch.float32, device=device)
        exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=device)
        steps = torch.zeros(n, dtype=torch.float32)
        has_state = np.zeros(n, bool)
        for i, p in enumerate(params):
            st = self.state.get(p)
            if not st:
                continue
            a, b = offset[i], offset[i + 1]
            exp_avg[a:b].copy_(st["exp_avg"].reshape(-1))
            exp_avg_sq[a:b].copy_(st["exp_avg_sq"].reshape(-1))
            steps[i] = float(st["step"])
            st["exp_avg"], st["exp_avg_sq"] = exp_avg[a:b].view_as(p), exp_avg_sq[a:b].view_as(p)
            st["step"] = steps[i]
            has_state[i] = True
        group_of = np.fromiter((gi for gi, g in enumerate(self.param_groups) for _ in g["params"]), np.int64, n)
        self._flat = dict(params=params, device=device, ptr=np.fromiter((p.data_ptr() for p in params), np.int64, n),
                          numel=numel, offset=offset, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, steps=steps,
                          steps_np=steps.numpy(), has_state=has_state, group_of=group_of,
                          grad_norm=torch.zeros((), dtype=torch.float32, device=device))

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if self._flat is None:
            self._flatten()
        c = self._flat
        params, n = c["params"], len(c["params"])
        gptr, has = np.zeros(n, np.int64), np.zeros(n, bool)
        for i, p in enumerate(params):
            g = p.grad
            if g is not None:
                if g.is_sparse or not g.is_contiguous():
                    raise RuntimeError(f"parameter {i}: vidar_b200.optim.AdamW takes dense contiguous gradients")
                gptr[i], has[i] = g.data_ptr(), True
        # per-group hyperparameters, read at every step, spread over the parameters
        groups = self.param_groups
        for g in groups:
            if g.get("amsgrad") or g.get("maximize"):
                raise RuntimeError("vidar_b200.optim.AdamW implements neither amsgrad nor maximize")
        gv = np.array([(g["lr"], g["weight_decay"], g["betas"][0], g["betas"][1], g["eps"]) for g in groups],
                      np.float64)[c["group_of"]]
        lr, wd, beta1, beta2, eps = gv.T
        steps = c["steps_np"]
        steps[has] += 1
        new = has & ~c["has_state"]
        for i in np.flatnonzero(new):            # first step of a parameter: torch's state, as views
            p, a, b = params[i], c["offset"][i], c["offset"][i + 1]
            self.state[p] = dict(step=c["steps"][i], exp_avg=c["exp_avg"][a:b].view_as(p),
                                 exp_avg_sq=c["exp_avg_sq"][a:b].view_as(p))
        c["has_state"] |= new
        # torch's scalars, in double from each parameter's own step count, then fp32 as its kernels take them
        # (a skipped parameter's scalars are not used.)  Python's pow, not numpy's, which differs in the last bit for
        # some powers; there are few distinct (beta1, beta2, step) -- usually one
        step = np.maximum(steps, 1).astype(np.float64)
        uniq, inv = np.unique(np.stack([beta1, beta2, step], 1), axis=0, return_inverse=True)
        bc = np.array([(1 - b1 ** s, (1 - b2 ** s) ** 0.5) for b1, b2, s in uniq.tolist()])[inv.reshape(-1)]
        scal = np.empty((n, 7), np.float32)
        scal[:, 0] = 1 - lr * wd
        scal[:, 1] = -(lr / bc[:, 0])
        scal[:, 2] = np.float32(1) / bc[:, 1].astype(np.float32)
        scal[:, 3] = 1 - beta1
        scal[:, 4] = beta2
        scal[:, 5] = 1 - beta2
        scal[:, 6] = eps
        clip = self.max_grad_norm is not None
        device = c["device"]
        if has.any():
            with torch.cuda.device(device):
                _lib.check(_lib.lib().vidar_adamw_step(
                    c["ptr"].ctypes.data, gptr.ctypes.data, c["numel"].ctypes.data, scal.ctypes.data, n,
                    _lib.ptr(c["exp_avg"]), _lib.ptr(c["exp_avg_sq"]), c["exp_avg"].numel(), int(clip),
                    float(self.max_grad_norm or 0.0), _lib.ptr(c["grad_norm"]), _lib.stream_ptr(device)))
        elif clip:
            c["grad_norm"].zero_()
        self.grad_norm = c["grad_norm"] if clip else None
        return loss

