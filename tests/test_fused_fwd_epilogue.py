"""GPU: the fused forward's epilogue -- bins resolved per 8-column chunk, dz staged in shared memory and written by TMA.

The walks over a thread's columns take a chunk without a bin lookup when it lies in the running bin, so these tests
put bin boundaries at every offset inside a chunk, on the CTA edges (columns 319/320, 639/640, 959/960), and make bins
of one and two columns, at G = 6 and at C = 1280.  dz leaves through TMA stores of 128-byte column boxes whose tensor
map clips columns >= C and rows >= N: the padding columns [C, ldd) must keep what was there, a ragged last tile must
not spill into the next rows, and a group that walks several row tiles refills the stages the stores read from.
The fused route is compared with the materialised route (GEMM -> fp32 logits -> grouped CE), and the plain
softmax-CE entry point (bags_ce_fwd) with a float64 restatement.
"""
import numpy as np
import pytest
import torch

from balancedgroupsoftmax_b200 import _native as nat

pytestmark = pytest.mark.gpu

K = 256
TOL = {   # as in test_gpu_parity.py
    torch.float32: dict(loss=1e-3, grad=1e-3),
    torch.bfloat16: dict(loss=2e-3, grad=5e-3),
}
SENTINEL = -7.0   # exact in bf16 and fp32


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _tables(starts, C, classes=300, seed=0):
    """DeviceTables with bins [starts[g], starts[g + 1]) tiling [0, C) and a random in-bin target per class."""
    from balancedgroupsoftmax_b200 import ops
    lens = [e - s for s, e in zip(starts, list(starts[1:]) + [C])]
    assert min(lens) >= 1
    rng = np.random.default_rng(seed)
    l2b = np.stack([rng.integers(0, n, classes) for n in lens]).astype(np.int32)
    flat = [v for s, n in zip(starts, lens) for v in (s, n)]
    dev = torch.device('cuda', 0)
    return ops.DeviceTables(len(starts), classes, C, torch.from_numpy(l2b).to(dev),
                            torch.zeros(classes, dtype=torch.int32, device=dev), nat.int32_array(flat),
                            np.array(list(zip(starts, lens)), dtype=np.int64))


def _operands(n, C, mode, weights, G, classes, seed):
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.relu(torch.randn(n, K, generator=g, device=dev)).to(mode)
    w = (torch.randn(C, K, generator=g, device=dev) * 0.1).to(mode)
    b = torch.randn(C, generator=g, device=dev) * 0.1
    labels = torch.randint(0, classes, (n,), generator=g, device=dev)
    if weights == 'u8':
        wm = (torch.rand(G, n, generator=g, device=dev) < 0.7).to(torch.uint8)
        avg = wm.float().sum(1).clamp_min(1.0)
    else:
        wm = torch.rand(G, n, generator=g, device=dev) * 2.0
        avg = wm.sum(1).clamp_min(1.0)
    return x, w, b, labels, wm, avg


def _fused_into(dz, x, w, b, labels, dt, wm, avg, colsum=None, lse=None):
    """bags_fwd on the fused route, writing into the given dz (so that its padding columns can be checked)."""
    from balancedgroupsoftmax_b200 import ops
    N, Kx = x.shape
    loss = torch.empty(dt.G, dtype=torch.float32, device=x.device)
    wm, wcode = ops._weights_arg(wm)
    ws = ops._workspace(x.device)
    nat.check(nat.lib().bags_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), b.data_ptr(), labels.data_ptr(), dt.label2bin.data_ptr(),
        dt.slices_host, wm.data_ptr(), wcode, avg.data_ptr(), N, Kx, dt.num_logits, dt.G, dt.num_classes,
        ops._dtype_code(x.dtype), None, 0, loss.data_ptr(), nat.ptr(lse), dz.data_ptr(), dz.stride(0), nat.ptr(colsum),
        colsum.shape[0] if colsum is not None else 0, ws.data_ptr(), ws.numel(), None, 0,
        ops._stream_ptr(x.device)), 'bags_fwd')
    return loss


def _check_bins(starts, C, mode, weights, n, want_colsum, seed=0):
    from balancedgroupsoftmax_b200 import ops
    dt = _tables(starts, C, seed=seed)
    assert ops.fused_eligible(dt)
    x, w, b, labels, wm, avg = _operands(n, C, mode, weights, dt.G, dt.num_classes, seed)
    ldd = ops.pad_cols(C) if C % 64 else C + 64
    dz = torch.full((n, ldd), SENTINEL, dtype=mode, device=x.device)
    lse = torch.empty((n, dt.G), dtype=torch.float32, device=x.device)
    colsum = torch.empty(((n + 127) // 128, C), dtype=torch.float32, device=x.device) if want_colsum else None
    loss = _fused_into(dz, x, w, b, labels, dt, wm, avg, colsum, lse)
    loss_m, _, lse_m, dz_m, colsum_m = ops.fused_fwd(x, w, b, labels, dt, wm, avg, want_lse=True, materialize=True,
                                                     want_colsum=want_colsum)
    torch.cuda.synchronize()
    tol = TOL[mode]
    for gi in range(dt.G):
        lf, lm = loss[gi].item(), loss_m[gi].item()
        assert abs(lf - lm) <= tol['loss'] * max(abs(lm), 1e-2), (gi, lf, lm)
    assert _rel(lse, lse_m) <= 1e-6
    assert _rel(dz[:, :C].float(), dz_m[:, :C].float()) <= tol['grad']
    # every column, including the one-column bins, on its own
    err = (dz[:, :C].double() - dz_m[:, :C].double()).abs().amax(0)
    scale = dz_m[:, :C].double().abs().amax(0).clamp_min(1e-3)
    assert (err / scale).max().item() <= 20 * tol['grad'], int((err / scale).argmax())
    assert bool((dz[:, C:] == SENTINEL).all()), 'dz padding columns were written'
    if want_colsum:
        assert _rel(colsum.sum(0), colsum_m.sum(0)) <= tol['grad']
    tail = slice(n - n % 128 or n - 128, n)
    assert _rel(dz[tail, :C].float(), dz_m[tail, :C].float()) <= tol['grad']


TABLES = {
    # one- and two-column bins, boundaries on the CTA edges 320 / 640 / 960, C = 1280
    'edges': ([0, 1, 3, 320, 640, 960], 1280),
    # boundaries one column before / after the CTA edges, a two-column bin across 319/320, a last bin of one column
    'around_edges': ([0, 319, 321, 639, 959, 1279], 1280),
}
for _o in range(1, 8):   # all five boundaries at offset o inside their 8-column chunk
    TABLES['offset%d' % _o] = ([0] + [8 * j + _o for j in (3, 41, 80, 120, 150)], 1236)


@pytest.mark.parametrize('name', sorted(TABLES))
def test_bin_boundaries(name):
    starts, C = TABLES[name]
    _check_bins(starts, C, torch.bfloat16, 'u8', 4096 + 77, want_colsum=True)


@pytest.mark.parametrize('weights', ['u8', 'f32'])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('want_colsum', [False, True], ids=['no_colsum', 'colsum'])
def test_operands_and_weights(mode, weights, want_colsum):
    _check_bins(TABLES['around_edges'][0], 1280, mode, weights, 2048 + 77, want_colsum, seed=1)


def test_stage_reuse_across_row_tiles():
    # every group walks 2-3 row tiles: the next tile's loads refill the stages the previous tile's dz stores read
    _check_bins(TABLES['offset3'][0], 1236, torch.bfloat16, 'u8', 131072 + 77, want_colsum=True, seed=2)


@pytest.mark.parametrize('C', [7, 1231])
@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_ce_fwd(C, mode):
    from balancedgroupsoftmax_b200 import ops
    n = 1024 + 77
    x, w, b, labels, wm, avg = _operands(n, C, mode, 'f32', 1, C, seed=C)
    wt, avg = wm[0].contiguous(), avg[:1].contiguous()
    ldd = ops.pad_cols(C)
    dz = torch.full((n, ldd), SENTINEL, dtype=mode, device=x.device)
    colsum = torch.empty(((n + 127) // 128, C), dtype=torch.float32, device=x.device)
    loss = torch.empty(1, dtype=torch.float32, device=x.device)
    ws = ops._workspace(x.device)
    nat.check(nat.lib().bags_ce_fwd(
        x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), b.data_ptr(), labels.data_ptr(), wt.data_ptr(),
        avg.data_ptr(), n, K, C, ops._dtype_code(mode), loss.data_ptr(), None, dz.data_ptr(), ldd, colsum.data_ptr(),
        colsum.shape[0], ws.data_ptr(), ws.numel(), None, 0, ops._stream_ptr(x.device)), 'bags_ce_fwd')
    torch.cuda.synchronize()
    z = x.double() @ w.double().t() + b.double()
    p = torch.softmax(z, 1)
    coef = wt.double() / avg.double()
    ref_loss = (coef * (torch.logsumexp(z, 1) - z.gather(1, labels[:, None])[:, 0])).sum()
    onehot = torch.nn.functional.one_hot(labels, C).double()
    ref_dz = (p - onehot) * coef[:, None]
    tol = TOL[torch.bfloat16]   # fp32 operands enter the tensor cores as TF32
    assert abs(loss.item() - ref_loss.item()) <= tol['loss'] * abs(ref_loss.item())
    assert _rel(dz[:, :C], ref_dz) <= tol['grad']
    assert bool((dz[:, C:] == SENTINEL).all()), 'dz padding columns were written'
    assert _rel(colsum.sum(0), dz[:, :C].double().sum(0)) <= tol['grad']   # sums of the stored values


def test_repeated_launches_are_bit_identical():
    from balancedgroupsoftmax_b200 import ops
    starts, C = TABLES['around_edges']
    dt = _tables(starts, C, seed=3)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 2 * (sms // 4) * 128 + 77   # groups loop over row tiles
    x, w, b, labels, wm, avg = _operands(n, C, torch.bfloat16, 'u8', dt.G, dt.num_classes, 3)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    runs = []
    with torch.cuda.stream(stream):
        for _ in range(3):
            loss, _, lse, dz, colsum = ops.fused_fwd(x, w, b, labels, dt, wm, avg, want_lse=True, want_colsum=True)
            runs.append((loss.clone(), lse.clone(), dz.clone(), colsum.clone()))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            out = ops.fused_fwd(x, w, b, labels, dt, wm, avg, want_lse=True, want_colsum=True)
        for _ in range(4):
            graph.replay()
            runs.append((out[0].clone(), out[2].clone(), out[3].clone(), out[4].clone()))
    stream.synchronize()
    loss0, lse0, dz0, cs0 = runs[0]
    for i, (loss, lse, dz, cs) in enumerate(runs[1:], 1):
        assert torch.equal(dz[:, :C], dz0[:, :C]), i
        assert torch.equal(lse, lse0), i
        assert torch.equal(cs, cs0), i
        assert torch.allclose(loss, loss0, rtol=1e-6, atol=0.0), (i, loss, loss0)
