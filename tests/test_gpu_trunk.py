"""GPU: the head's trunk on this library's wgmma GEMMs -- shared FCs (Linear + ReLU) and fc_reg
(convfc_bbox_head.py:138-143,167) through LinearActFunction, forward and backward, against plain torch fp32 (the numerics
reference for a floating-point kernel: fp32 nn.Linear + ReLU + autograd on the CPU)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('N,K,C,relu', [(1024, 12544, 1024, True), (1000, 1024, 1024, True), (517, 1024, 4924, False),
                                        (3, 64, 1024, True), (130, 1024, 4, False)])
def test_linear_act_forward_backward_vs_torch(N, K, C, relu, mode):
    from balancedgroupsoftmax_b200 import ops
    g = torch.Generator().manual_seed(N + K + C)
    x = torch.randn(N, K, generator=g)
    W = torch.randn(C, K, generator=g) * (1.0 / K ** 0.5)
    b = torch.randn(C, generator=g) * 0.1
    dy = torch.randn(N, C, generator=g)
    xd = x.cuda().requires_grad_(True)
    Wd = torch.nn.Parameter(W.cuda())
    bd = torch.nn.Parameter(b.cuda())
    out_dtype = torch.float32 if (mode == torch.float32 or not relu) else torch.bfloat16
    y = ops.LinearActFunction.apply(xd, Wd, bd, relu, mode, out_dtype)
    y.backward(dy.cuda().to(y.dtype))
    torch.cuda.synchronize()
    # reference: fp32 torch on the CPU.  ReLU is discontinuous: an output within rounding distance of zero may land on the
    # other side in TF32 / bf16, and each flipped mask entry changes the gradients by O(1) -- so the reference backward
    # uses THIS run's mask (checked separately below to agree with the fp32 one wherever the fp32 output is clearly
    # away from zero), which makes the gradient comparison a test of the three contractions, not of the mask's luck.
    xr, Wr, br = x.clone().requires_grad_(True), W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    lin = torch.nn.functional.linear(xr, Wr, br)
    mask = (y.detach().float().cpu() > 0).float() if relu else torch.ones_like(lin)
    yr = lin * mask
    yr.backward(dy.to(y.dtype).float())
    tol = 2e-3 if mode == torch.float32 else 1.2e-2      # TF32 / bf16 operand rounding, fp32 accumulation
    assert y.dtype == out_dtype and rel(y.float(), torch.relu(lin) if relu else lin) <= tol
    errs = dict(dW=rel(Wd.grad, Wr.grad), db=rel(bd.grad, br.grad), dX=rel(xd.grad, xr.grad))
    assert max(errs.values()) <= tol, errs
    if relu:
        assert bool((y >= 0).all())
        far = lin.detach().abs() > (0.02 if mode == torch.float32 else 0.1)
        assert torch.equal((y.float().cpu() > 0)[far], (lin.detach() > 0)[far])


def test_bf16_weight_copy_follows_parameter_updates():
    from balancedgroupsoftmax_b200 import ops
    W = torch.nn.Parameter(torch.randn(64, 128, device='cuda'))
    x = torch.randn(8, 128, device='cuda')
    y0 = ops.LinearActFunction.apply(x, W, None, False, torch.bfloat16, torch.float32)
    y1 = ops.LinearActFunction.apply(x, W, None, False, torch.bfloat16, torch.float32)
    assert torch.equal(y0, y1)
    with torch.no_grad():
        W.mul_(2.0)                                     # what an optimizer step does: in place, version counter moves
    y2 = ops.LinearActFunction.apply(x, W, None, False, torch.bfloat16, torch.float32)
    assert rel(y2, 2.0 * y0) < 1e-6


def test_head_trunk_runs_native_and_matches_torch_trunk():
    """GSBBoxHeadWith0.forward with the native trunk vs the same module's nn.Linear trunk (native_trunk=False)."""
    from balancedgroupsoftmax_b200.head import GSBBoxHeadWith0
    from balancedgroupsoftmax_b200.tables import synthetic_tables
    t = synthetic_tables(1231, seed=0)

    def make(native):
        torch.manual_seed(0)
        h = GSBBoxHeadWith0(num_fcs=2, in_channels=16, fc_out_channels=256, roi_feat_size=4, num_classes=1231,
                            gs_config=dict(tables=t, others_sample_ratio=8.0, num_bins=5, compute_dtype='fp32',
                                           native_trunk=native,
                                           loss_bin=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0)))
        h.init_weights()
        return h.cuda().train()
    a, b = make(True), make(False)
    feats = torch.randn(200, 16, 4, 4, device='cuda')
    labels = torch.zeros(200, dtype=torch.long, device='cuda')
    labels[:50] = torch.randint(1, 1231, (50,), device='cuda')
    outs = []
    for h in (a, b):
        cls, reg = h(feats)
        torch.manual_seed(1)
        h._sample_calls = 0
        losses = h.loss(cls, reg, labels, None, torch.randn(200, 4, device='cuda'), torch.ones(200, 4, device='cuda'))
        sum(losses.values()).backward()
        outs.append((cls.x_cls.float(), reg.float(), h.shared_fcs[0].weight.grad, h.fc_reg.weight.grad))
    # forward values agree to TF32 rounding; the gradients additionally see the few ReLU mask entries that rounding flips
    for i, (u, v) in enumerate(zip(*outs)):
        assert rel(u, v) <= (3e-3 if i < 2 else 3e-2), (i, rel(u, v))
