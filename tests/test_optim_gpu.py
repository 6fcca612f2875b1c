"""The configs' optimizer step (vidar_b200/optim.py, csrc/optim.cu) against torch: clip_grad_norm_ then
torch.optim.AdamW(foreach=False), and an fp64 restatement of both, over 10 steps of a list with odd numels, 1- and
0-element tensors, more tensors than one launch's table holds, three groups with their own lr and weight decay and
one tensor without a gradient on some steps, with the clip active and inactive.  Then non-finite gradients (alone and
under a GradScaler), determinism, launches and host syncs, state dicts both ways with torch.optim.AdamW, and the
pre-training step with `pretrain.config_optimizer`."""
import io

import pytest
import torch

pytestmark = pytest.mark.gpu

TABLE = 896                  # tensors per launch (csrc/optim.cu kTable)
GROUPS = [dict(lr=1e-3, weight_decay=0.01), dict(lr=3e-4, weight_decay=0.0), dict(lr=2e-3, weight_decay=0.1)]


def _numels(many):
    big = [1, 0, 7, 1000003, 1, 33, 4099, 0, 65537, 2, 257 * 129]
    if not many:
        return big
    g = torch.Generator().manual_seed(7)
    return big + torch.randint(0, 300, (TABLE + 40,), generator=g).tolist()


def _params(numels, cuda, seed=0):
    g = torch.Generator(device=cuda).manual_seed(seed)
    return [torch.nn.Parameter(torch.randn(n, generator=g, device=cuda) * 0.5) for n in numels]


def _groups(params):
    return [dict(params=params[k::3], **GROUPS[k]) for k in range(3)]


def _grads(numels, cuda, step, scale):
    """Per-step gradients; parameter 3 has none on steps 2 and 5."""
    g = torch.Generator(device=cuda).manual_seed(100 + step)
    out = [torch.randn(n, generator=g, device=cuda) * scale for n in numels]
    if step in (2, 5):
        out[3] = None
    return out


def _set(params, grads):
    for p, g in zip(params, grads):
        p.grad = None if g is None else g.clone()


class _Fp64:
    """clip_grad_norm_ + torch's single-tensor AdamW restated in fp64."""

    def __init__(self, params, max_norm):
        self.p = [p.detach().double().clone() for p in params]
        self.m = [torch.zeros_like(p) for p in self.p]
        self.v = [torch.zeros_like(p) for p in self.p]
        self.t = [0] * len(self.p)
        self.hyper = [GROUPS[i % 3] for i in range(len(self.p))]
        self.max_norm = max_norm

    def step(self, grads):
        gs = [None if g is None else g.double() for g in grads]
        norm = torch.sqrt(sum((g * g).sum() for g in gs if g is not None))
        coef = min(self.max_norm / (float(norm) + 1e-6), 1.0) if self.max_norm else 1.0
        for i, g in enumerate(gs):
            if g is None:
                continue
            h, g = self.hyper[i], g * coef
            self.t[i] += 1
            self.p[i] *= 1 - h["lr"] * h["weight_decay"]
            self.m[i] = self.m[i] * 0.9 + 0.1 * g
            self.v[i] = self.v[i] * 0.999 + 0.001 * g * g
            bc1, bc2 = 1 - 0.9 ** self.t[i], 1 - 0.999 ** self.t[i]
            self.p[i] -= h["lr"] / bc1 * self.m[i] / (self.v[i].sqrt() / bc2 ** 0.5 + 1e-8)
        return float(norm)


def _torch_step(opt, params, max_norm):
    norm = None
    if max_norm:
        norm = torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], max_norm)
    opt.step()
    return norm


def _ulps(a, b):
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max()) if a.numel() else 0


@pytest.mark.parametrize("max_norm", [1.0, 1e6], ids=["clip_active", "clip_inactive"])
def test_ten_steps_match_torch_and_fp64(cuda, max_norm):
    from vidar_b200 import _lib, optim
    numels = _numels(True)
    ours_p, ref_p = _params(numels, cuda), _params(numels, cuda)
    f64 = _Fp64(ref_p, max_norm)
    ours = optim.AdamW(_groups(ours_p), max_grad_norm=max_norm)
    ref = torch.optim.AdamW(_groups(ref_p), foreach=False)
    worst_ulp = 0
    for step in range(10):
        grads = _grads(numels, cuda, step, 0.05)
        _set(ours_p, grads)
        _set(ref_p, grads)
        n0 = _lib.launch_count()
        ours.step()
        assert _lib.launch_count() - n0 == 4                # two tables: a norm and an update launch each
        ref_norm = _torch_step(ref, ref_p, max_norm)
        norm64 = f64.step(grads)
        assert abs(float(ours.grad_norm) - float(ref_norm)) <= 1e-6 * float(ref_norm)
        assert abs(float(ours.grad_norm) - norm64) <= 1e-6 * norm64
        if step == 0:
            assert (max_norm / norm64 < 1) == (max_norm == 1.0)     # the clip is active in one case only
    for i, (a, b) in enumerate(zip(ours_p, ref_p)):
        if a.numel() == 0:
            continue
        sa, sb = ours.state[a], ref.state[b]
        assert float(sa["step"]) == float(sb["step"]) == (8 if i == 3 else 10)
        for x, y, z in ((a.detach(), b.detach(), f64.p[i]), (sa["exp_avg"], sb["exp_avg"], f64.m[i]),
                        (sa["exp_avg_sq"], sb["exp_avg_sq"], f64.v[i])):
            scale = float(y.abs().max())
            assert float((x - y).abs().max()) <= 1e-6 * scale, i
            e_ours, e_torch = float((x.double() - z).abs().max()), float((y.double() - z).abs().max())
            assert e_ours <= 2 * e_torch + 1e-7, (i, e_ours, e_torch)
            worst_ulp = max(worst_ulp, _ulps(x, y))
    print(f"max_norm {max_norm}: largest ulp difference from torch {worst_ulp}")


@pytest.mark.parametrize("bad", ["inf", "nan"])
def test_non_finite_gradients_match_torch(cuda, bad):
    from vidar_b200 import optim
    numels = [5, 1000, 3]
    ours_p, ref_p = _params(numels, cuda, 1), _params(numels, cuda, 1)
    ours = optim.AdamW(ours_p, lr=1e-3, max_grad_norm=35)
    ref = torch.optim.AdamW(ref_p, lr=1e-3, foreach=False)
    for step in range(2):
        grads = _grads(numels, cuda, step, 1.0)
        if step == 1:
            grads[1][[3, 500]] = float(bad)
        _set(ours_p, grads)
        _set(ref_p, grads)
        ours.step()
        _torch_step(ref, ref_p, 35)
    for a, b, g in zip(ours_p, ref_p, grads):
        a, b = a.detach(), b.detach()
        assert torch.equal(a.isnan(), b.isnan())
        want = torch.ones_like(a, dtype=torch.bool) if bad == "nan" else g.isinf()
        assert torch.equal(a.isnan(), want)
        fin = ~b.isnan()
        torch.testing.assert_close(a[fin], b[fin], rtol=0, atol=1e-6 * float(b[fin].abs().max()) if fin.any() else 0)
    assert ours.grad_norm.isinf() if bad == "inf" else ours.grad_norm.isnan()


def test_grad_scaler_skips_a_step_with_an_inf_gradient(cuda):
    from vidar_b200 import optim
    numels = [5, 1000, 0, 3]
    ps = _params(numels, cuda, 2)
    opt = optim.AdamW(ps, lr=1e-3, max_grad_norm=35)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
    grads = _grads(numels, cuda, 0, 1024.0)
    _set(ps, grads)
    scaler.scale(torch.zeros((), device=cuda))          # what a training step's scaler.scale(loss) sets up
    scaler.step(opt)
    scaler.update()
    before = [p.detach().clone() for p in ps]
    state = {k: v.clone() for k, v in opt.state[ps[1]].items()}
    grads = _grads(numels, cuda, 1, 1024.0)
    grads[1][7] = float("inf")
    _set(ps, grads)
    scaler.scale(torch.zeros((), device=cuda))
    scaler.step(opt)
    scaler.update()
    assert all(torch.equal(a, b) for a, b in zip(ps, before))
    assert all(torch.equal(v, opt.state[ps[1]][k]) for k, v in state.items())
    assert scaler.get_scale() == 512.0


def test_same_gradients_give_bitwise_the_same_parameters(cuda):
    from vidar_b200 import optim
    numels = _numels(False)
    runs = []
    for _ in range(2):
        ps = _params(numels, cuda, 3)
        opt = optim.AdamW(_groups(ps), max_grad_norm=1.0)
        for step in range(3):
            _set(ps, _grads(numels, cuda, step, 0.1))
            opt.step()
        runs.append(([p.detach().clone() for p in ps], opt.grad_norm.clone()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    assert torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("clip", [True, False])
def test_two_launches_and_no_host_sync(cuda, clip):
    from vidar_b200 import _lib, optim
    numels = _numels(False)
    ps = _params(numels, cuda, 4)
    opt = optim.AdamW(_groups(ps), max_grad_norm=35 if clip else None)
    for step in range(2):                     # the first step makes the state, the second reuses it
        _set(ps, _grads(numels, cuda, step, 0.1))
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        torch.cuda.set_sync_debug_mode("error")
        try:
            opt.step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert _lib.launch_count() - n0 == (2 if clip else 1)
    assert (opt.grad_norm is not None) == clip


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


@pytest.mark.parametrize("direction", ["ours_to_torch", "torch_to_ours"])
def test_state_dicts_interoperate_with_torch(cuda, direction):
    from vidar_b200 import optim
    numels = _numels(False)
    make = {"ours": lambda ps: optim.AdamW(_groups(ps), max_grad_norm=1.0),
            "torch": lambda ps: torch.optim.AdamW(_groups(ps), foreach=False)}
    first, second = direction.split("_to_")
    ps1 = _params(numels, cuda, 5)
    o1 = make[first](ps1)
    for step in range(3):
        _set(ps1, _grads(numels, cuda, step, 0.1))
        o1.step() if first == "ours" else _torch_step(o1, ps1, 1.0)
    ps2 = [torch.nn.Parameter(p.detach().clone()) for p in ps1]
    o2 = make[second](ps2)
    o2.load_state_dict(_roundtrip(o1.state_dict()))
    if second == "ours":
        assert all(o2.state[p]["exp_avg"].untyped_storage().data_ptr() == o2._flat["exp_avg"].untyped_storage().data_ptr()
                   for p in ps2 if p in o2.state)
    for step in range(3, 6):
        grads = _grads(numels, cuda, step, 0.1)
        for ps, o, kind in ((ps1, o1, first), (ps2, o2, second)):
            _set(ps, grads)
            o.step() if kind == "ours" else _torch_step(o, ps, 1.0)
    for a, b in zip(ps1, ps2):
        if a.numel():
            assert float((a - b).abs().max()) <= 1e-6 * float(a.detach().abs().max())
            assert float(o1.state[a]["step"]) == float(o2.state[b]["step"])


def test_pretrain_step_with_the_config_optimizer(cuda):
    """Two `train_step`s with `config_optimizer` against torch's AdamW over the same `paramwise_groups` after
    clip_grad_norm_(35), fed the gradients the step computed; the backbone moves at a tenth of the rate."""
    from vidar_b200 import optim, pretrain
    small = dict(encoder_layers=3, decoder_layers=2, future_frames=2, bev_hw=(40, 40), ray_grid_num=64)
    model, _ = pretrain.build(cuda, None, seed=1, **small)
    sample = pretrain.synthetic_sample(cuda, frames=2, img_hw=(96, 160), rays_per_frame=800, future_frames=2,
                                       bev_hw=(40, 40))
    opt = pretrain.config_optimizer(model)
    names = [n for n, _ in model.named_parameters()]
    start = [p.detach().clone() for p in model.parameters()]
    ref_p = [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in model.parameters()]
    ref_groups = [dict(g, params=[ref_p[i]]) for i, g in enumerate(optim.paramwise_groups(model, 2e-4, 0.01,
                                                                                        {"backbone": dict(lr_mult=0.1)}))]
    ref = torch.optim.AdamW(ref_groups, lr=2e-4, weight_decay=0.01, foreach=False)
    captured = []
    opt.register_step_pre_hook(lambda o, a, k: captured.append([None if p.grad is None else p.grad.clone()
                                                                 for p in model.parameters()]))
    for step in range(2):
        loss, stages = pretrain.train_step(model, opt, sample, None, record=True)
        assert torch.isfinite(loss) and "optimizer" in [s for s, _ in stages]
        _set(ref_p, captured[-1])
        _torch_step(ref, [p for p in ref_p if p.requires_grad], 35.0)
        if step == 0:
            for name, p, p0 in zip(names, model.parameters(), start):
                if p.requires_grad:
                    moved = float((p.detach() - p0).abs().max())
                    lr = 2e-5 if name.startswith("backbone.") else 2e-4
                    # Adam's first step moves an element by at most lr, plus the decay lr * wd * |p|
                    assert moved <= 1.001 * lr * (1 + 0.01 * float(p0.abs().max())), (name, moved)
            for name, p, group in zip(names, model.parameters(), opt.param_groups):
                assert group["params"][0] is p
                assert group["lr"] == pytest.approx(2e-5 if name.startswith("backbone.") and p.requires_grad else 2e-4)
    assert len(captured) == 2
    for name, a, b in zip(names, model.parameters(), ref_p):
        assert float((a.detach() - b.detach()).abs().max()) <= 1e-6 * float(b.detach().abs().max()), name
