"""-m gpu: the row-shard entries of the glue and the heads against the rows of their whole-tensor siblings, bitwise.

  af2_embed_pair_init_rows  rows [row0, row0 + rows) of af2_embed_pair_init's x, and its whole m   (seq_index with gaps)
  af2_recycle_embed_rows    rows of af2_recycle_embed's x (from the same rows of x and of the previous pair), its whole m
  af2_distogram_head_rows   rows of af2_distogram_head's output from x_rows and the same rows as columns, x_cols
  af2_angle_heads_rows      rows of af2_angle_heads' theta / phi / omega, both omega modes

Windows start at 0, at offsets that are not multiples of 8 and end at N; N is not always a multiple of 8.  Every malformed
call returns AF2_ERR_BAD_ARG, launches nothing and leaves its NaN-filled outputs untouched."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BAD_ARG = -1


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib.load()


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _windows(n: int):
    return [(0, n), (0, 5), (3, min(n, 14)), (n - 7, n), (9, n - 2)]


def _rejected(fn, args, outs):
    lib = _lib()
    for o in outs:
        o.fill_(float("nan"))
    torch.cuda.synchronize()
    n0 = lib.af2_launch_count()
    rc = getattr(lib, fn)(*args, _ops()._stream_ptr())
    torch.cuda.synchronize()
    assert rc == BAD_ARG, (fn, rc)
    assert lib.af2_launch_count() == n0, f"{fn}: a rejected call launched a kernel"
    for o in outs:
        assert torch.isnan(o).all(), f"{fn}: a rejected call wrote its output"


@pytest.mark.parametrize("d", [128, 256])
@pytest.mark.parametrize("n", [21, 32])
def test_distogram_head_rows_bitwise(d, n):
    ops = _ops()
    torch.manual_seed(d + n)
    x = torch.randn(n, n, d, device="cuda")
    g, be = 1 + 0.1 * torch.randn(d, device="cuda"), 0.1 * torch.randn(d, device="cuda")
    w, b = torch.randn(37, d, device="cuda") / d ** 0.5, torch.randn(37, device="cuda")
    whole = ops.distogram_head(x[None], g, be, w, b)
    for r0, r1 in _windows(n):
        out = ops.distogram_head_rows(x[r0:r1].contiguous(), x[:, r0:r1].contiguous(), g, be, w, b)
        assert _same(out, whole[:, r0:r1]), (r0, r1)


@pytest.mark.parametrize("d", [32, 128, 320])
@pytest.mark.parametrize("n", [19, 24])
@pytest.mark.parametrize("sym", [False, True])
def test_angle_heads_rows_bitwise(d, n, sym):
    ops = _ops()
    torch.manual_seed(d + n + sym)
    lins = [torch.nn.Linear(d, k).cuda() for k in (25, 13, 25)]
    assert ops.angle_heads_ok(d, (25, 13, 25))
    pk = ops.pack_angle_heads(lins[0].weight, lins[0].bias, lins[1].weight, lins[1].bias, lins[2].weight, lins[2].bias)
    x = torch.randn(n, n, d, device="cuda")
    whole = ops.angle_heads(pk, x[None], sym)
    for r0, r1 in _windows(n):
        rows = ops.angle_heads_rows(pk, x[r0:r1].contiguous(), x[:, r0:r1].contiguous() if sym else None, sym)
        for name, got, ref in zip(("theta", "phi", "omega"), rows, whole):
            assert _same(got, ref[:, r0:r1]), (name, r0, r1)


def _pair_init_inputs(n, S, d, R=4):
    torch.manual_seed(n + d)
    vocab = 22
    seq = torch.randint(0, vocab, (1, n), device="cuda")
    msa = torch.randint(0, vocab, (1, S, n), device="cuda")
    emb, wp, bp = torch.randn(vocab, d, device="cuda"), torch.randn(2 * d, d, device="cuda") / d ** 0.5, torch.randn(2 * d, device="cuda")
    pos = torch.randn(2 * R + 1, d, device="cuda")
    # gaps beyond +-R on both sides of the diagonal, not monotonic
    idx = torch.cat([torch.arange(0, n // 2) * 3, torch.arange(n - n // 2) + 200])
    idx[1], idx[2] = idx[2].item(), idx[1].item()
    return seq, msa, emb, wp, bp, pos, R, idx.cuda()


@pytest.mark.parametrize("n,d", [(21, 32), (24, 128)])
def test_embed_pair_init_rows_bitwise(n, d):
    ops = _ops()
    seq, msa, emb, wp, bp, pos, R, idx = _pair_init_inputs(n, 3, d)
    x, m = ops.embed_pair_init(seq, msa, emb, wp, bp, pos, R, seq_index=idx, m_rows=5)
    for r0, r1 in _windows(n):
        xr, mr = ops.embed_pair_init_rows(seq, msa, emb, wp, bp, pos, R, r0, r1 - r0, seq_index=idx, m_rows=5)
        assert _same(xr, x[:, r0:r1]), (r0, r1)
        assert _same(mr[:, :3], m[:, :3]), (r0, r1)


@pytest.mark.parametrize("n,d", [(21, 64), (24, 256)])
def test_recycle_embed_rows_bitwise(n, d):
    ops = _ops()
    torch.manual_seed(n * d)
    x0, m0 = torch.randn(1, n, n, d, device="cuda"), torch.randn(1, 3, n, d, device="cuda")
    coords, single, pair = torch.randn(1, n, 3, device="cuda") * 6, torch.randn(1, n, d, device="cuda"), torch.randn(1, n, n, d, device="cuda")
    p = [1 + 0.1 * torch.randn(d, device="cuda"), 0.1 * torch.randn(d, device="cuda"), 1 + 0.1 * torch.randn(d, device="cuda"),
         0.1 * torch.randn(d, device="cuda"), torch.randn(32, d, device="cuda")]
    x, m = ops.recycle_embed_(x0.clone(), m0.clone(), coords, single, pair, *p)
    for r0, r1 in _windows(n):
        xr, mr = ops.recycle_embed_rows_(x0[:, r0:r1].clone(), m0.clone(), coords, single, pair[:, r0:r1].contiguous(), *p, r0)
        assert _same(xr, x[:, r0:r1]), (r0, r1)
        assert _same(mr, m), (r0, r1)


def test_rows_entries_reject_malformed_calls():
    n, d, rows = 20, 128, 6
    dev = "cuda"
    f = lambda *s: torch.empty(*s, device=dev)  # noqa: E731
    x_rows, x_cols = torch.randn(rows + 4, n, d, device=dev), torch.randn(n, rows + 4, d, device=dev)
    g, be, w, b = f(d), f(d), f(37, d), f(37)
    out = f(rows + 4, n, 37)
    # distogram: null x_cols, bad dim, more rows than n
    P = lambda t: t.data_ptr()  # noqa: E731
    for args in [(P(x_rows), None, P(g), P(be), P(w), P(b), P(out), rows, n, d, 37),
                 (P(x_rows), P(x_cols), P(g), P(be), P(w), P(b), P(out), rows, n, 96, 37),
                 (P(x_rows), P(x_cols), P(g), P(be), P(w), P(b), P(out), n + 1, n, d, 37),
                 (P(x_rows), P(x_cols), P(g), P(be), P(w), P(b), P(out), -1, n, d, 37)]:
        _rejected("af2_distogram_head_rows", args, [out])
    # angle heads: null x_cols with symmetrize, rows > n, bad dim, buckets that do not fit
    planes, bias = torch.zeros(d // 32 * 3 * 64 * 32, dtype=torch.bfloat16, device=dev), f(64)
    th, ph, om = f(rows + 4, n, 25), f(rows + 4, n, 13), f(rows + 4, n, 25)
    outs = [th, ph, om]
    base = (P(x_rows), P(x_cols), P(planes), P(bias), P(th), P(ph), P(om))
    for args in [(P(x_rows), None) + base[2:] + (rows, n, d, 25, 13, 25, 1),
                 base + (n + 1, n, d, 25, 13, 25, 0),
                 base + (-2, n, d, 25, 13, 25, 1),
                 base + (rows, n, 48, 25, 13, 25, 0),
                 base + (rows, n, d, 30, 30, 30, 0)]:
        _rejected("af2_angle_heads_rows", args, outs)
    # pair init: windows outside [0, n), bad dim
    seq, msa = torch.zeros(1, n, dtype=torch.int64, device=dev), torch.zeros(1, 2, n, dtype=torch.int64, device=dev)
    emb, wp, bp, pos = f(22, d), f(2 * d, d), f(2 * d), f(9, d)
    xo, mo = f(1, rows + 4, n, d), f(1, 2, n, d)
    ws = torch.empty(_lib().af2_embed_pair_init_workspace(1, n, d), dtype=torch.uint8, device=dev)
    head = (P(seq), P(msa), P(emb), 22, None, None, P(wp), P(bp), P(pos), 4, None, P(xo), P(mo), 1, 2, n)
    for tail in [(d, n - rows + 1, rows), (d, -1, rows), (d, 0, -1), (d, 0, n + 1), (130, 0, rows)]:
        _rejected("af2_embed_pair_init_rows", head + tail + (P(ws), ws.numel()), [xo, mo])
    # recycling: windows outside [0, n), misaligned x
    coords, single, pp = f(1, n, 3), f(1, n, d), f(1, rows + 4, n, d)
    tbl, bnd = f(32, d), f(32)
    xr, mr = f(1, rows + 4, n, d), f(1, 2, n, d)
    for xp, r0, rr in [(P(xr), n - rows + 1, rows), (P(xr), -1, rows), (P(xr), 0, n + 1), (P(xr) + 4, 0, rows)]:
        args = (P(coords), 3, P(single), P(pp), P(g), P(be), P(g), P(be), P(tbl), P(bnd), 32, xp, P(mr), n * d, 1, n, d, 1e-5, r0, rr)
        _rejected("af2_recycle_embed_rows", args, [xr, mr])
