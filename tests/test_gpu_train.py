"""The tail of a training step on the GPU: flat Adam (stmp_adam_flat) against torch.optim.Adam, eager and CUDA-graph replayed,
and the weight-gradient contraction (stmp_dcrnn_bwd_wgrad) against a float64 contraction of the same operands."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, distributed as D, ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None


def _models(seed):
    torch.manual_seed(seed)
    a = torch.nn.Sequential(torch.nn.Linear(7, 13), torch.nn.Tanh(), torch.nn.Linear(13, 3)).to(DEV)
    b = torch.nn.Sequential(torch.nn.Linear(7, 13), torch.nn.Tanh(), torch.nn.Linear(13, 3)).to(DEV)
    b.load_state_dict(a.state_dict())
    return a, b


@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_flat_adam_matches_torch_adam(wd):
    a, b = _models(0)
    sync = D.FlatGradSync(a.parameters())
    opt_a = D.FlatAdam(sync, lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    opt_b = torch.optim.Adam(b.parameters(), lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    c0 = _lib.path_counters().get("k_adam_flat", 0)
    for it in range(12):
        x = torch.randn(32, 7, device=DEV)
        a(x).square().mean().backward()
        opt_a.step()
        opt_b.zero_grad()
        b(x).square().mean().backward()
        opt_b.step()
        assert float(sync.flat.abs().max()) == 0.0                      # the gradient buffer is cleared in the same launch
    assert _lib.path_counters()["k_adam_flat"] == c0 + 12
    assert float(opt_a.step_count) == 12.0
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert pa.data_ptr() >= opt_a.flat.data_ptr() and pa.data_ptr() < opt_a.flat.data_ptr() + opt_a.flat.numel() * 4
        torch.testing.assert_close(pa, pb, rtol=2e-5, atol=1e-6)


def test_flat_adam_cuda_graph_replay_counts_steps_on_device():
    a, b = _models(1)
    sync = D.FlatGradSync(a.parameters())
    opt_a = D.FlatAdam(sync, lr=3e-3)
    opt_b = torch.optim.Adam(b.parameters(), lr=3e-3)
    x = torch.randn(16, 7, device=DEV)

    def body():
        a(x).square().mean().backward()
        opt_a.step()

    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    steps = int(float(opt_a.step_count))
    for _ in range(steps):
        opt_b.zero_grad()
        b(x).square().mean().backward()
        opt_b.step()
    assert steps == 6                                                    # eager warm-up + 5 replays; the capture itself runs nothing
    for pa, pb in zip(a.parameters(), b.parameters()):
        torch.testing.assert_close(pa, pb, rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize("tc", [0, 1])
@pytest.mark.parametrize("cin,rows", [(2, 12 * 5 * 207), (1, 1000), (4, 207 * 3 + 5), (2, 7)])
def test_dcrnn_wgrad_vs_float64(cin, rows, tc):
    """tc = 1: the wgmma contraction (TF32 hi/lo split, K-major operands); tc = 0: the fp32 FFMA kernel."""
    _lib.set_option("dcrnn_wgrad_tc", tc)
    try:
        _wgrad_case(cin, rows, "k_dcrnn_wgrad_tc" if tc else "k_dcrnn_wgrad")
    finally:
        _lib.set_option("dcrnn_wgrad_tc", WGRAD_TC_DEFAULT)


def test_dcrnn_wgrad_small_gradients_keep_their_precision():
    """d pre-activations of a mean loss are ~1e-6: the operand split must not lose them (an fp16 split would flush them to subnormals)."""
    _lib.set_option("dcrnn_wgrad_tc", 1)
    try:
        _wgrad_case(2, 4 * 207, "k_dcrnn_wgrad_tc", dp_scale=1e-6)
    finally:
        _lib.set_option("dcrnn_wgrad_tc", WGRAD_TC_DEFAULT)


WGRAD_TC_DEFAULT = 1


def _wgrad_case(cin, rows, kernel, dp_scale=1.0):
    torch.manual_seed(cin)
    Co, K = 32, 2
    C = cin + Co
    ld = ops.dcrnn_bwd_basis_ld(cin, Co, K)
    S1 = torch.full((rows, 1, ld), float("nan"), device=DEV)            # pad columns hold garbage: they must never reach a result
    S2 = torch.full((rows, 1, ld), float("nan"), device=DEV)
    S1[..., :3 * C] = torch.randn(rows, 1, 3 * C, device=DEV)
    S2[..., :3 * C] = torch.randn(rows, 1, 3 * C, device=DEV)
    dpzr = torch.randn(rows, 2 * Co, device=DEV) * dp_scale
    dph = torch.randn(rows, Co, device=DEV) * dp_scale
    c0 = _lib.path_counters().get(kernel, 0)
    gz, gr, gh, gbz, gbr, gbh = ops.dcrnn_bwd_wgrad(cin, K, S1, S2, dpzr, dph, True)
    assert _lib.path_counters().get(kernel, 0) == c0 + 1
    s1, s2 = S1[:, 0, :3 * C].double(), S2[:, 0, :3 * C].double()
    dWzr, dWh = s1.t() @ dpzr.double(), s2.t() @ dph.double()

    def unstack(d):                                                      # stacked block 0 -> W[0,0] and W[1,0]; block 1 + o -> W[o,1]
        blk = d.view(3, C, Co)
        return torch.stack([torch.stack([blk[0], blk[1]]), torch.stack([blk[0], blk[2]])])

    scale = (rows ** 0.5) * dp_scale
    for got, ref in ((gz, unstack(dWzr[:, :Co])), (gr, unstack(dWzr[:, Co:])), (gh, unstack(dWh))):
        assert got.shape == (2, K, C, Co)
        assert float((got.double() - ref).abs().max()) < 2e-6 * scale * 4
    for got, ref in ((gbz, dpzr[:, :Co].double().sum(0)), (gbr, dpzr[:, Co:].double().sum(0)), (gbh, dph.double().sum(0))):
        assert float((got.double() - ref).abs().max()) < 2e-6 * scale * 4
    # deterministic: same bits on a second call
    again = ops.dcrnn_bwd_wgrad(cin, K, S1, S2, dpzr, dph, True)
    assert torch.equal(again[0], gz) and torch.equal(again[2], gh) and torch.equal(again[5], gbh)
