"""The association of every weight-gradient reduce.  Each fused training path computes its weight gradients as per-CTA partials in a
workspace and then a fixed-order sum of them (`fixed_order_sum`, csrc/rows.cuh): warp w of 8 adds parts [w·per, (w+1)·per), per =
⌈parts/8⌉, in two interleaved accumulators with an odd tail into the first, and the 8 warp sums are added left to right.  That order is
what makes repeated backwards bit-identical and a power-of-two loss scale exact, so it is pinned here bit for bit: each C entry is
called on seeded random operands with a workspace the test owns, and every dw / db / dpeep element is recomputed in float32 from the
partials the contraction left there.  Part counts follow from the launches: min(SMs, ⌈rows/16⌉) for the TF32 contraction, min(2·SMs,
⌈rows/16⌉) for the FFMA one, min(2·SMs, ⌈rows/32⌉) for the 64-wide GConvGRU one and rows_grid(rows) for the LSTM peephole partials."""
import pytest
import torch

from pytorch_geometric_temporal_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
PARTS = [0, 1, 7, 8, 9, "full"]          # 0: rows = 0; "full": as many parts as the launch allows, more tiles than parts
NAN = float("nan")


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _rows(parts, tile, cap):
    """Rows that make `parts` partials (at most `cap`) of `tile`-row tiles, the last tile ragged."""
    if parts == 0:
        return 0
    if parts == "full":
        return tile * cap * 2 + 7
    return tile * parts - 5


def _parts(rows, tile, cap):
    return min(cap, (rows + tile - 1) // tile)


def _fixed_order_sum(P):
    """The reduce kernels' sum over the n parts of P (n, M), in float32, in their association."""
    n, M = P.shape
    per = (n + 7) // 8
    subs = []
    for w in range(8):
        q, q1 = w * per, min(w * per + per, n)
        s0, s1 = torch.zeros(M), torch.zeros(M)
        while q + 2 <= q1:
            s0, s1 = s0 + P[q], s1 + P[q + 1]
            q += 2
        if q < q1:
            s0 = s0 + P[q]
        subs.append(s0 + s1)
    t = subs[0]
    for s in subs[1:]:
        t = t + s
    return t


def _sum(P, src):
    """fixed_order_sum of P's columns `src` (any shape) -> a tensor of src's shape."""
    return _fixed_order_sum(P[:, src.reshape(-1)]).view(src.shape)


def _randn(*shape):
    return torch.randn(*shape, device=DEV)


def _operands(rows, *widths):
    """Seeded random (rows, width) operands; at least one row, so that rows = 0 still passes non-NULL pointers."""
    return [_randn(max(rows, 1), w) for w in widths]


def _workspace(nbytes):
    return torch.zeros(int(nbytes) // 4, device=DEV)


def _check(rc):
    assert rc == _lib.STMP_OK, _lib.last_error()
    torch.cuda.synchronize()


def _equal(got, want):
    got = got.cpu()
    assert got.shape == want.shape
    assert torch.equal(got, want), f"{int((got != want).sum())} of {got.numel()} elements differ"


def _gate_src(MG8, m, gate, o):
    """Column of a k_dcrnn_wgrad<32> / k_dcrnn_wgrad_tc partial holding output channel o of gate 0 (z), 1 (r) or 2 (h) for basis column
    m: S1ᵀ[dpz | dpr] at m·64 + gate·32 + o, then S2ᵀdph at MG8·64 + m·32 + o."""
    return torch.where(gate == 2, MG8 * 64 + m * 32 + o, m * 64 + gate * 32 + o)


def _ar(n):
    return torch.arange(n)


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("tc", [1, 0])
def test_dcrnn_bwd_wgrad(tc, parts, bias):
    """stmp_dcrnn_bwd_wgrad with the TF32 contraction (k_dcrnn_wgrad_tc) or the FFMA one (k_dcrnn_wgrad<32>), then
    k_dcrnn_wgrad_reduce into the (2, K, C, 32) weights of each gate."""
    torch.manual_seed(1)
    cin, K, C = 2, 2, 34
    ld = ops.dcrnn_bwd_basis_ld(cin, 32, K)
    cap = _sms() if tc else 2 * _sms()
    rows = _rows(parts, 16, cap)
    S1, S2, dpzr, dph = _operands(rows, ld, ld, 64, 32)
    ws = _workspace(_lib.lib().stmp_dcrnn_bwd_wgrad_workspace_bytes(cin))
    g = torch.full((3, 2, K, C, 32), NAN, device=DEV)
    gb = torch.full((3, 32), NAN, device=DEV)
    bs = [_lib.ptr(gb[i]) if bias else None for i in range(3)]
    kernel = "k_dcrnn_wgrad_tc" if tc else "k_dcrnn_wgrad"
    _lib.set_option("dcrnn_wgrad_tc", tc)
    try:
        c0 = _lib.path_counters().get(kernel, 0)
        _check(_lib.lib().stmp_dcrnn_bwd_wgrad(cin, 32, K, rows, ld, _lib.ptr(S1), _lib.ptr(S2), _lib.ptr(dpzr), _lib.ptr(dph), _lib.ptr(ws),
                                               _lib.ptr(g[0]), _lib.ptr(g[1]), _lib.ptr(g[2]), *bs, _lib.stream_ptr()))
        assert _lib.path_counters().get(kernel, 0) == c0 + int(rows > 0)
    finally:
        _lib.set_option("dcrnn_wgrad_tc", 1)
    n, stride = _parts(rows, 16, cap), ld * 96 + 96
    P = ws[:n * stride].view(n, stride).cpu()
    o, k, c, j = torch.meshgrid(_ar(2), _ar(K), _ar(C), _ar(32), indexing="ij")
    m = torch.where(k == 0, 0, 1 + o) * C + c                         # block 0 feeds W[0,0] and W[1,0]; block 1 + o feeds W[o,1]
    for gate in range(3):
        _equal(g[gate], _sum(P, _gate_src(ld, m, torch.full_like(m, gate), j)))
    if bias:
        _equal(gb, _sum(P, ld * 96 + _ar(96).view(3, 32)))
    else:
        assert torch.isnan(gb).all()


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("parts", PARTS)
def test_gru_bwd_wgrad(parts, bias):
    """stmp_gru_bwd_wgrad: k_dcrnn_wgrad_tc, then k_gru_wgrad_reduce into the forward's dwcat [96][112], zero where the layout has no
    basis column (absent operators, absent X channels, padding)."""
    torch.manual_seed(2)
    n_ops, cin = 1, 3
    C, nb = cin + 32, n_ops + 1
    ld = ops.gru_bwd_basis_ld(n_ops, cin)
    cap = _sms()
    rows = _rows(parts, 16, cap)
    S1, S2, dpzr, dph = _operands(rows, ld, ld, 64, 32)
    ws = _workspace(_lib.lib().stmp_gru_bwd_wgrad_workspace_bytes(n_ops, cin))
    dw = torch.full((96, 112), NAN, device=DEV)
    db = torch.full((96,), NAN, device=DEV)
    _check(_lib.lib().stmp_gru_bwd_wgrad(n_ops, cin, rows, ld, _lib.ptr(S1), _lib.ptr(S2), _lib.ptr(dpzr), _lib.ptr(dph), _lib.ptr(ws),
                                         _lib.ptr(dw), _lib.ptr(db) if bias else None, _lib.stream_ptr()))
    n, stride = _parts(rows, 16, cap), ld * 96 + 96
    P = ws[:n * stride].view(n, stride).cpu()
    row, col = torch.meshgrid(_ar(96), _ar(112), indexing="ij")
    hcol = col < 96                                                    # columns H | Op0 H | Op1 H, then X | Op0 X | Op1 X | pad
    blk = torch.where(hcol, col // 32, (col - 96) // 4)
    c = torch.where(hcol, cin + col % 32, (col - 96) % 4)
    zero = (blk >= nb) | (~hcol & (c >= cin))
    src = torch.where(zero, 0, _gate_src(ld, blk * C + c, row // 32, row % 32))
    _equal(dw, torch.where(zero, 0.0, _sum(P, src)))
    if bias:
        _equal(db, _sum(P, ld * 96 + _ar(96)))
    else:
        assert torch.isnan(db).all()


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("cout", [32, 64])
def test_gru_rows_wgrad(cout, parts, bias):
    """stmp_gru_rows_wgrad (k_dcrnn_wgrad<32>, then k_gru_rows_wgrad_reduce) and stmp_gru_wide_rows_wgrad (k_gru_wide_rows_wgrad, one
    partial per (gate, CTA), then k_gru_wide_rows_wgrad_reduce) into the packed dw [3 cout][nb] and db [3 cout]."""
    torch.manual_seed(3)
    n_ops, cin = 1, 5
    nb = (n_ops + 1) * (cin + cout)
    ld = ops.gru_rows_basis_ld(n_ops, cin, cout)
    tile = 16 if cout == 32 else 32
    cap = 2 * _sms()
    rows = _rows(parts, tile, cap)
    S1, S2, dpzr, dph = _operands(rows, ld, ld, 2 * cout, cout)
    name = "stmp_gru_rows_" if cout == 32 else "stmp_gru_wide_rows_"
    ws = _workspace(getattr(_lib.lib(), name + "wgrad_workspace_bytes")(n_ops, cin))
    dw = torch.full((3 * cout, nb), NAN, device=DEV)
    db = torch.full((3 * cout,), NAN, device=DEV)
    _check(getattr(_lib.lib(), name + "wgrad")(n_ops, cin, rows, ld, _lib.ptr(S1), _lib.ptr(S2), _lib.ptr(dpzr), _lib.ptr(dph), _lib.ptr(ws),
                                                _lib.ptr(dw), _lib.ptr(db) if bias else None, _lib.stream_ptr()))
    n = _parts(rows, tile, cap)
    row, m = torch.meshgrid(_ar(3 * cout), _ar(nb), indexing="ij")
    if cout == 32:
        stride = ld * 96 + 96
        P = ws[:n * stride].view(n, stride).cpu()
        want_w, want_b = _sum(P, _gate_src(ld, m, row // 32, row % 32)), _sum(P, ld * 96 + _ar(96))
    else:                                                              # partial [gate][part][ld·64 + 64]: Sᵀ·dpre_gate, then its column sums
        stride = ld * 64 + 64
        P = ws[:3 * n * stride].view(3, n, stride).cpu()
        want_w = torch.cat([_sum(P[g], m[:64] * 64 + row[:64]) for g in range(3)])
        want_b = torch.cat([_sum(P[g], ld * 64 + _ar(64)) for g in range(3)])
    _equal(dw, want_w)
    if bias:
        _equal(db, want_b)
    else:
        assert torch.isnan(db).all()


@pytest.mark.parametrize("peep", [True, False])
@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("parts", PARTS)
@pytest.mark.parametrize("variant", [_lib.LSTM_GCONV, _lib.LSTM_GC])
def test_lstm_rows_wgrad(variant, parts, bias, peep):
    """stmp_lstm_rows_wgrad: k_dcrnn_wgrad<64>, then k_lstm_rows_wgrad_reduce into dw [128][nb], db [128] and, from the per-CTA peephole
    sums k_lstm_rows_bwd_a leaves in the scratch behind its N·48 floats, dpeep [96]."""
    torch.manual_seed(4 + variant)
    n_ops, cin = 1, 5
    nb, ld = ops.lstm_rows_nb(variant, n_ops, cin), ops.lstm_rows_basis_ld(variant, n_ops, cin)
    cap = 2 * _sms()
    rows = _rows(parts, 16, cap)
    n = _parts(rows, 16, cap)                                          # = rows_grid(rows) for rows > 0: both count 16-row tiles up to 2·SMs
    S, = _operands(rows, ld)
    dpre = _randn(2, max(rows, 1), 64)
    scratch = _randn(rows * 48 + max(n, 1) * 96)
    ws = _workspace(_lib.lib().stmp_lstm_rows_wgrad_workspace_bytes(variant, n_ops, cin))
    dw = torch.full((128, nb), NAN, device=DEV)
    db = torch.full((128,), NAN, device=DEV)
    dpeep = torch.full((96,), NAN, device=DEV)
    _check(_lib.lib().stmp_lstm_rows_wgrad(variant, n_ops, cin, rows, ld, _lib.ptr(S), _lib.ptr(dpre), _lib.ptr(scratch), _lib.ptr(ws),
                                           _lib.ptr(dw), _lib.ptr(db) if bias else None, _lib.ptr(dpeep) if peep else None,
                                           _lib.stream_ptr()))
    stride = ld * 128 + 128
    P = ws[:n * stride].view(n, stride).cpu()
    row, m = torch.meshgrid(_ar(128), _ar(nb), indexing="ij")          # Sᵀ[dpi | dpf] at m·64 + row, then Sᵀ[dpc | dpo]
    _equal(dw, _sum(P, torch.where(row < 64, m * 64 + row, ld * 64 + m * 64 + row - 64)))
    if bias:
        _equal(db, _sum(P, ld * 128 + _ar(128)))
    else:
        assert torch.isnan(db).all()
    if peep:
        _equal(dpeep, _sum(scratch[rows * 48:rows * 48 + n * 96].view(n, 96).cpu(), _ar(96)))
    else:
        assert torch.isnan(dpeep).all()
