"""Modulated deformable convolution (vidar_b200/dcn.py, csrc/dcn.cu) on the GPU: the output and all five gradients
against the fp64 oracle on every kernel path (16-byte and scalar channel loops, 3xTF32 and cuBLAS GEMMs, one and
several column chunks, stride / padding / dilation / non-square kernels), the reference's two layer shapes against
torchvision in fp64, the DCN backbone against the same backbone on torchvision's fp32 op, and the pre-training step."""
import copy
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import dcn_ref
from tests.parity import close

pytestmark = pytest.mark.gpu


def _inputs(dev, N, C, H, W, O, k=(3, 3), stride=(1, 1), padding=(1, 1), dilation=(1, 1), offset_std=3.0, bias=True,
            seed=0):
    g = torch.Generator().manual_seed(seed)
    kh, kw = k
    Ho = (H + 2 * padding[0] - (dilation[0] * (kh - 1) + 1)) // stride[0] + 1
    Wo = (W + 2 * padding[1] - (dilation[1] * (kw - 1) + 1)) // stride[1] + 1
    x = torch.randn(N, C, H, W, generator=g)
    off = torch.randn(N, 2 * kh * kw, Ho, Wo, generator=g) * offset_std
    mask = torch.rand(N, kh * kw, Ho, Wo, generator=g)
    w = torch.randn(O, C, kh, kw, generator=g) / (C * kh * kw) ** 0.5
    b = torch.randn(O, generator=g) if bias else None
    gy = torch.randn(N, O, Ho, Wo, generator=g)
    return [t.to(dev) if t is not None else None for t in (x, off, mask, w, b, gy)]


def _kink_free(off, stride, padding, dilation, k, eps=1e-4):
    """[N, 2K, Ho, Wo] bool: the coordinate of this offset channel is farther than eps px from every integer line
    (where d/d(h, w) of the bilinear form jumps and either one-sided value is legitimate) and from the range ends."""
    kh, kw = k
    N, _, Ho, Wo = off.shape
    o = off.detach().double().cpu().view(N, kh * kw, 2, Ho, Wo)
    i = torch.arange(kh).repeat_interleave(kw).double()
    j = torch.arange(kw).repeat(kh).double()
    h = (torch.arange(Ho).double()[None, :] * stride[0] - padding[0] + i[:, None] * dilation[0])[None, :, :, None] + o[:, :, 0]
    w = (torch.arange(Wo).double()[None, :] * stride[1] - padding[1] + j[:, None] * dilation[1])[None, :, None, :] + o[:, :, 1]
    ok = lambda t: (t - t.round()).abs() > eps
    both = ok(h) & ok(w)
    return torch.stack([both, both], 2).view(N, 2 * kh * kw, Ho, Wo)


def _check_against_oracle(dev, **case):
    from vidar_b200.dcn import modulated_deform_conv2d
    stride, padding, dilation = (case.get(k, (1, 1)) for k in ("stride", "padding", "dilation"))
    x, off, mask, w, b, gy = _inputs(dev, **case)
    leaves = [t.clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, w, b)]
    y = modulated_deform_conv2d(*leaves, stride, padding, dilation, 1, 1)
    assert y.is_contiguous(memory_format=torch.channels_last)
    y.backward(gy)
    y_ref, grads = dcn_ref.deform_conv2d_backward(x, off, mask, w, b, gy, stride, padding, dilation)
    close(y, y_ref, "out")
    keep_off = _kink_free(off, stride, padding, dilation, case.get("k", (3, 3)))
    for what, leaf, ref in zip(("input", "offset", "mask", "weight", "bias"), leaves, grads):
        if leaf is None:
            continue
        close(leaf.grad, ref, f"grad_{what}", keep=keep_off if what == "offset" else None)


CASES = {
    # C % 4 == 0 and kh*kw*C, Cout multiples of 128: 16-byte sampling loops; the 3xTF32 GEMM for grad_cols, and for
    # the forward too when kh*kw*C <= dcn.TC_MAX_K (C = 64: K = 576 is not a multiple of 128, so a 1x1 kernel is used)
    "vec4_tc": dict(N=2, C=128, H=10, W=13, O=128),
    "vec4_tc_fwd": dict(N=2, C=256, H=10, W=13, O=128, k=(1, 1), padding=(0, 0)),
    # C % 4 != 0: scalar loops; the GEMMs on cuBLAS
    "scalar_cublas": dict(N=2, C=5, H=9, W=11, O=7, bias=False),
    # C % 4 == 0 but kh*kw*C not a multiple of 128: 16-byte loops, cuBLAS
    "vec4_cublas": dict(N=1, C=16, H=12, W=9, O=8),
    "stride2": dict(N=2, C=128, H=11, W=14, O=128, stride=(2, 2)),
    "pad0_dil2": dict(N=1, C=64, H=14, W=12, O=128, padding=(0, 0), dilation=(2, 2), bias=False),
    "nonsquare": dict(N=1, C=12, H=9, W=15, O=6, k=(2, 3), stride=(2, 1), padding=(1, 0), dilation=(1, 2)),
    "small_offsets": dict(N=2, C=128, H=8, W=8, O=128, offset_std=0.6),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_oracle(cuda, name):
    _check_against_oracle(cuda, **CASES[name])


@pytest.mark.parametrize("tc", [True, False])
def test_batch_over_several_column_chunks(cuda, monkeypatch, tc):
    """5 images in chunks of 2 (+ the remainder 1): every chunk's rows, gradients and weight-gradient sum."""
    from vidar_b200 import dcn
    C, H, W = (128, 7, 9) if tc else (8, 7, 9)
    per_image = H * W * 9 * C
    monkeypatch.setattr(dcn, "MAX_COLS_BYTES", 2 * 4 * per_image + 100)
    assert dcn.chunk_images(5, per_image) == 2
    _check_against_oracle(cuda, N=5, C=C, H=H, W=W, O=128 if tc else 12)


def test_chunk_bound_keeps_one_image_when_an_image_is_larger():
    from vidar_b200 import dcn
    assert dcn.chunk_images(6, dcn.MAX_COLS_BYTES) == 1
    assert dcn.chunk_images(6, 58 * 100 * 9 * 256) == 6          # a stage-3 layer of the reference input: one chunk


@pytest.mark.parametrize("stage", [3, 4])
def test_reference_layer_shape_matches_torchvision_fp64(cuda, stage):
    """6 x 256 x 58 x 100 -> 256 (layer3) and 6 x 512 x 29 x 50 -> 512 (layer4), the backbone's DCN layers at the
    6 x 928 x 1600 input, with bias=False as the backbone builds them.  Every output and gradient is within the max-norm
    bar of tests/parity.py; its L2 error is within that bar too, or -- where a sum over K = 9 * 512 terms that cancel
    leaves more fp32 rounding than the bar allows -- within 3x the L2 error of torchvision's own fp32 op."""
    import torchvision
    from vidar_b200.dcn import modulated_deform_conv2d
    C, H, W = (256, 58, 100) if stage == 3 else (512, 29, 50)
    x, off, mask, w, _, gy = _inputs(cuda, 6, C, H, W, C, offset_std=2.0, bias=False, seed=stage)
    keep = _kink_free(off, (1, 1), (1, 1), (1, 1), (3, 3)).to(cuda)
    runs = []
    for impl, dt in (("ours", torch.float32), ("torchvision", torch.float32), ("torchvision", torch.float64)):
        leaves = [t.detach().to(dt).clone().requires_grad_(True) for t in (x, off, mask, w)]
        if impl == "ours":
            y = modulated_deform_conv2d(*leaves, None, 1, 1, 1, 1, 1)
        else:
            y = torchvision.ops.deform_conv2d(leaves[0], leaves[1], leaves[3], None, padding=1, mask=leaves[2])
        y.backward(gy.to(dt))
        g_off = leaves[1].grad.masked_fill(~keep, 0)
        runs.append([y.detach().double()] + [t.grad.double() for t in leaves[:1]] + [g_off.double()] +
                    [t.grad.double() for t in leaves[2:]])
        del y, leaves
    ours, tv32, ref = runs
    for what, a, t, r in zip(("out", "grad_input", "grad_offset", "grad_mask", "grad_weight"), ours, tv32, ref):
        _close_or_like_fp32(a, t, r, what)


def _close_or_like_fp32(a, t, r, what, factor=3):
    """`a` against the fp64 result `r`: within the norms of tests/parity.py, or no farther from `r` than `factor` x the
    fp32 result `t` of torchvision is (max and L2 norms)."""
    a, t, r = (v.detach().double().cpu() for v in (a, t, r))
    assert torch.isfinite(a).all(), what
    for norm, bar in ((lambda v: v.abs().max().item(), 1e-4), (lambda v: v.norm().item(), 2e-5)):
        err, err_tv = norm(a - r), norm(t - r)
        assert err <= max(bar * norm(r), factor * err_tv), f"{what}: err {err:.3e}, torchvision fp32 {err_tv:.3e}, |ref| {norm(r):.3e}"


def _torchvision_pack_forward(self, x):
    import torchvision
    out = self.conv_offset(x)
    o1, o2, mask = torch.chunk(out, 3, dim=1)
    return torchvision.ops.deform_conv2d(x, torch.cat((o1, o2), 1), self.weight, self.bias, stride=self.stride,
                                         padding=self.padding, dilation=self.dilation, mask=torch.sigmoid(mask))


def test_dcn_backbone_matches_torchvision_backbone(cuda, monkeypatch):
    """C3-C5 and every layer3 / layer4 parameter gradient of ImageBackbone(dcn=True) against the same backbone with each
    DCN on torchvision's op, run in fp32 and in fp64: ours is as close to the fp64 run as the parity norms ask, or
    within 3x of torchvision's fp32 run: 26 stacked layers amplify fp32 rounding in both."""
    from vidar_b200.dcn import ModulatedDeformConv2dPack
    from vidar_b200.pretrain import ImageBackbone
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    torch.manual_seed(0)
    ours = ImageBackbone(dcn=True)
    g = torch.Generator().manual_seed(1)
    for m in ours.modules():
        # offsets of about half a pixel from the bias, a data-dependent part of ~0.1 px from the weight, masks away
        # from 0.5.  A sample whose coordinate crosses an integer line between two runs changes grad_offset by a jump;
        # with offsets that move ~1 px with the activations, the rounding of any fp32 run crosses many of them and the
        # gradients of all three runs scatter far beyond fp32 rounding, so the data-dependent part is kept small.
        if isinstance(m, ModulatedDeformConv2dPack):
            m.conv_offset.weight.data.copy_(torch.randn(m.conv_offset.weight.shape, generator=g) * 1e-3)
            m.conv_offset.bias.data.copy_(torch.randn(m.conv_offset.bias.shape, generator=g) * 0.5)
    tv32 = copy.deepcopy(ours)
    for m in tv32.modules():
        if isinstance(m, ModulatedDeformConv2dPack):
            m.forward = _torchvision_pack_forward.__get__(m)
    tv64 = copy.deepcopy(tv32).double()
    img = torch.randn(2, 3, 96, 160, generator=g, dtype=torch.float64).to(cuda)
    outs = []
    for model in (ours, tv32, tv64):
        model.to(cuda).train()
        feats = model(img.to(next(model.parameters()).dtype))
        sum((f * torch.linspace(-1, 1, f.numel(), device=cuda, dtype=f.dtype).view_as(f)).sum() for f in feats).backward()
        grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if n.startswith(("layer3", "layer4"))}
        outs.append(([f.detach() for f in feats], grads))
    (fa, ga), (ft, gt), (fr, gr) = outs
    for lvl, a, t, r in zip(("C3", "C4", "C5"), fa, ft, fr):
        _close_or_like_fp32(a, t, r, lvl)
    assert set(ga) == set(gr) and sum("conv_offset" in n for n in ga) == 2 * 26
    for n in ga:
        _close_or_like_fp32(ga[n], gt[n], gr[n], n)


SMALL = dict(encoder_layers=2, decoder_layers=2, future_frames=2, bev_hw=(40, 40), ray_grid_num=64, dcn=True)
SAMPLE = dict(frames=2, img_hw=(96, 160), rays_per_frame=800, future_frames=2, bev_hw=(40, 40))


def run_reduced_pretrain_step(dev):
    """(model, loss) of one pre-training step of the SMALL model with the DCN backbone on a SAMPLE-sized input."""
    from vidar_b200 import pretrain
    from vidar_b200 import synthetic
    model, opt = pretrain.build(dev, None, seed=1, **SMALL)
    sample = pretrain.synthetic_sample(dev, **SAMPLE)
    # the rig's intrinsics are for the full image: scale its pixel rows to the small one so pillars project inside
    l2i = sample["lidar2img"].copy()
    l2i[..., 0, :] *= SAMPLE["img_hw"][1] / synthetic.IMG_HW[1]
    l2i[..., 1, :] *= SAMPLE["img_hw"][0] / synthetic.IMG_HW[0]
    sample["lidar2img"] = l2i
    loss, _ = pretrain.train_step(model, opt, sample, None)
    return model, loss


def test_pretrain_step_with_dcn(cuda):
    model, loss = run_reduced_pretrain_step(cuda)
    assert torch.isfinite(loss)
    offs = [(n, p) for n, p in model.named_parameters() if "conv_offset" in n]
    assert len(offs) == 2 * 26
    for n, p in offs:
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0, n


def test_status_codes_and_shape_errors(cuda):
    from vidar_b200 import _lib
    from vidar_b200.dcn import modulated_deform_conv2d
    x, off, mask, w, b, _ = _inputs(cuda, 2, 8, 6, 7, 4)
    with pytest.raises(ValueError, match="offset"):
        modulated_deform_conv2d(x, off[:, :-2], mask, w, b, 1, 1, 1, 1, 1)
    with pytest.raises(TypeError, match="float32"):
        modulated_deform_conv2d(x.double(), off, mask, w, b, 1, 1, 1, 1, 1)
    xl = x.permute(0, 2, 3, 1).contiguous()
    cols = torch.empty(6 * 7 * 9 * 8, device=cuda)
    L = _lib.lib()
    args = [_lib.ptr(xl), _lib.ptr(off), _lib.ptr(mask), _lib.ptr(cols), 2, 8, 6, 7, 6, 7, 3, 3, 1, 1, 1, 1, 1, 1]
    assert L.vidar_dcn_im2col(*args, 1, 2, _lib.stream_ptr(cuda)) == 1
    assert b"bad image range" in L.vidar_last_error()
    assert L.vidar_dcn_im2col(*args[:8], 5, 7, *args[10:], 1, 1, _lib.stream_ptr(cuda)) == 1
    assert b"does not match" in L.vidar_last_error()
    assert L.vidar_dcn_im2col(*args, 1, 1, _lib.stream_ptr(cuda)) == 0
    torch.cuda.synchronize()


def _sharded_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from vidar_b200 import pretrain, sharding
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    res = []
    for group in (None, dist.group.WORLD):
        model, opt = pretrain.build(dev, group, seed=1, **SMALL)
        sample = pretrain.synthetic_sample(dev, **SAMPLE)
        opt.zero_grad(set_to_none=True)
        loss = sum(model.forward_train(sample["img"], sample["lidar2img"], sample["gt_points"]).values())
        loss.backward()
        if group is not None:
            sharding.allreduce_partial_grads(model, group)
        res.append((float(loss), {n: p.grad.detach().cpu() for n, p in model.named_parameters() if p.grad is not None}))
    if rank == 0:
        torch.save(res, out)
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_dcn_step_equals_single_gpu(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "dcn.pt")
    mp.spawn(_sharded_worker, args=(2, 29040 + os.getpid() % 100, out), nprocs=2, join=True)
    (l1, g1), (l2, g2) = torch.load(out, weights_only=False)
    assert abs(l1 - l2) <= 1e-4 * abs(l1)
    assert set(g1) == set(g2)
    for n in g1:
        scale = float(g1[n].abs().max())
        torch.testing.assert_close(g2[n], g1[n], rtol=2e-3, atol=2e-4 * scale + 1e-9, msg=lambda m: f"{n}: {m}")
