"""GPU: the fused forward's persistent grid of CTA groups.

Four CTAs own a 128-row tile and exchange their softmax partials through the per-stream workspace; the grid holds at
most one group per four SMs, and each group walks the row tiles group, group + groups, ...  These tests cover a ragged
last tile, groups that loop over two or three row tiles (double-buffered exchange slots), a row count above the old
4096-CTA limit of the fused route, and repeated launches -- eager and graph replays -- on one workspace, whose arrival
counters are never reset.
"""
import pytest
import torch

from balancedgroupsoftmax_b200.tables import synthetic_tables

pytestmark = pytest.mark.gpu

K = 1024
TOL = {   # as in test_kernel_resources.py / test_gpu_parity.py
    torch.float32: dict(loss=1e-3, grad=1e-3),
    torch.bfloat16: dict(loss=2e-3, grad=5e-3),
}


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _problem(n, mode, seed):
    from balancedgroupsoftmax_b200 import ops
    dev = torch.device('cuda', 0)
    t = synthetic_tables(1231, seed=0)
    dt = ops.DeviceTables.from_tables(t, dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.relu(torch.randn(n, K, generator=g, device=dev)).to(mode)
    w = (torch.randn(t.num_logits, K, generator=g, device=dev) * 0.05).to(mode)
    b = torch.randn(t.num_logits, generator=g, device=dev) * 0.1
    labels = torch.zeros(n, dtype=torch.long, device=dev)
    labels[:n // 4] = torch.randint(1, t.num_classes, (n // 4,), generator=g, device=dev)
    wmask, avg = ops.sample_others(labels, dt, 8.0, seed)
    return dt, x, w, b, labels, wmask, avg


def _looping_rows():
    """Rows for which every CTA group walks at least two row tiles (one group three) on this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * (sms // 4) * 128 + 77


def _check_against_materialised(n, mode, seed=0):
    from balancedgroupsoftmax_b200 import ops
    dt, x, w, b, labels, wmask, avg = _problem(n, mode, seed)
    loss_f, logits_f, lse_f, dz_f, colsum_f = ops.fused_fwd(x, w, b, labels, dt, wmask, avg, want_lse=True,
                                                            want_colsum=True)
    loss_m, _, lse_m, dz_m, colsum_m = ops.fused_fwd(x, w, b, labels, dt, wmask, avg, want_lse=True,
                                                     materialize=True, want_colsum=True)
    torch.cuda.synchronize()
    assert logits_f is None   # the fused kernel ran
    assert colsum_f.shape[0] == (n + 127) // 128
    tol = TOL[mode]
    C = dt.num_logits
    for gi in range(dt.G):
        lf, lm = loss_f[gi].item(), loss_m[gi].item()
        assert abs(lf - lm) <= tol['loss'] * max(abs(lm), 1e-2), (gi, lf, lm)
    assert _rel(lse_f, lse_m) <= 1e-6
    assert _rel(dz_f[:, :C].float(), dz_m[:, :C].float()) <= tol['grad']
    assert _rel(colsum_f.sum(0), colsum_m.sum(0)) <= tol['grad']
    # the last, ragged tile on its own
    tail = slice(n - 77, n)
    assert _rel(lse_f[tail], lse_m[tail]) <= 1e-6
    assert _rel(dz_f[tail, :C].float(), dz_m[tail, :C].float()) <= tol['grad']


@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_ragged_last_tile(mode):
    _check_against_materialised(4096 + 77, mode)


@pytest.mark.parametrize('mode', [torch.float32, torch.bfloat16], ids=['fp32', 'bf16'])
def test_groups_loop_over_row_tiles(mode):
    _check_against_materialised(_looping_rows(), mode, seed=1)


def test_rows_above_old_grid_limit():
    # 4096 CTAs x 128 / 4 rows was the largest N the one-cluster-per-row-tile grid accepted
    _check_against_materialised(131072 + 77, torch.bfloat16, seed=2)


def test_repeated_launches_on_one_workspace():
    from balancedgroupsoftmax_b200 import ops
    n = _looping_rows()
    dt, x, w, b, labels, wmask, avg = _problem(n, torch.bfloat16, 3)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    runs = []
    with torch.cuda.stream(stream):   # eager calls and the captured graph share this stream's workspace
        for _ in range(3):
            loss, _, lse, dz, _ = ops.fused_fwd(x, w, b, labels, dt, wmask, avg, want_lse=True)
            runs.append((loss.clone(), lse.clone(), dz.clone()))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            out = ops.fused_fwd(x, w, b, labels, dt, wmask, avg, want_lse=True)
        for _ in range(4):
            graph.replay()
            runs.append((out[0].clone(), out[2].clone(), out[3].clone()))
    stream.synchronize()
    loss0, lse0, dz0 = runs[0]
    for i, (loss, lse, dz) in enumerate(runs[1:], 1):
        assert torch.equal(dz, dz0), i
        assert torch.equal(lse, lse0), i
        assert torch.allclose(loss, loss0, rtol=1e-6, atol=0.0), (i, loss, loss0)
