"""-m gpu: the row-shard entries of the structure module against their whole-tensor siblings, bitwise, in one process.

  af2_ipa_attention_rows           the query rows [row0, row0 + rows) of af2_ipa_attention, from those pair rows alone
  af2_structure_layer_rows_begin   with _end on the same workspace: af2_structure_layer, whether one call covers every row or
  / _end                           P row shards (uneven) are run one by one and their to_out rows concatenated
  ops.pair_projection_rows_        those rows of ops.pair_projection_ (bf16 and strict GEMMs, forced and planned bands)

Every malformed call of the new entries returns AF2_ERR_BAD_ARG (AF2_ERR_WORKSPACE for a workspace too small), launches
nothing and leaves its NaN-filled output untouched; the host wrappers raise ValueError on bad shapes before any call."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BAD_ARG = -1
WORKSPACE = -4
DEV = "cuda"


def _ops():
    from alphafold2_b200 import ops
    return ops


def _lib():
    from alphafold2_b200 import _lib
    return _lib.load()


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _frames(g, n):
    from oracle import structure_oracle as SO
    R = SO.quaternion_to_matrix(torch.randn(1, n, 4, generator=g, dtype=torch.float64)).float()
    return R.to(DEV).contiguous(), (torch.randn(1, n, 3, generator=g) * 5).to(DEV)


def _mask(n, kind):
    if kind == "none":
        return None
    m = torch.ones(1, n, dtype=torch.bool)
    if kind == "padded":
        m[0, n - max(1, n // 4):] = False              # padding: the last query rows are fully masked
    else:
        m[0, ::3] = False                              # scattered: fully masked query rows inside every window
    return m.to(DEV)


def _windows(n):
    r = max(1, n // 3)
    return sorted({(0, r), ((n - r) // 2, r), (n - r, r), (n // 2, 1)})


@pytest.mark.parametrize("d", [32, 128, 256])
@pytest.mark.parametrize("H", [1, 4, 8, 16])
@pytest.mark.parametrize("n", [1, 33, 257])
def test_ipa_attention_rows_bitwise(n, H, d):
    ops = _ops()
    g = torch.Generator().manual_seed(n * 1000 + H * 10 + d)
    proj = torch.randn(1, n, 84 * H, generator=g).to(DEV)
    pair = torch.randn(1, n, n, d, generator=g).to(DEV)
    R, t = _frames(g, n)
    wb = (torch.randn(H, d, generator=g) * d ** -0.5).to(DEV)
    bb, pw = torch.randn(H, generator=g).to(DEV), torch.randn(H, generator=g).to(DEV)
    for kind in ("none", "padded", "scattered"):
        mask = _mask(n, kind)
        whole = ops.ipa_attention(proj, pair, wb, bb, pw, mask, R, t, H)
        for row0, rows in _windows(n):
            got = ops.ipa_attention_rows(proj, pair[:, row0:row0 + rows].contiguous(), wb, bb, pw, mask, R, t, H, row0)
            assert _same(got, whole[:, row0:row0 + rows]), (kind, row0, rows)


def _layer_model(d, H, seed):
    """The packed weights of one structure layer with every parameter random (to_out included: attach zeroes it)."""
    import alphafold2_b200 as A
    torch.manual_seed(seed)
    model = A.attach_structure_module(A.Alphafold2(dim=d, depth=1, heads=2, dim_head=16, predict_coords=True,
                                                   structure_module_heads=H))
    with torch.no_grad():
        for p in model.ipa_block.parameters():
            p.copy_(torch.randn_like(p) * p.shape[-1] ** -0.5)
    return model.to(DEV).eval()


def _layer_inputs(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    single = torch.randn(1, n, d, generator=g).to(DEV)
    pair = torch.randn(1, n, n, d, generator=g).to(DEV)
    q = torch.randn(1, n, 4, generator=g)
    q = torch.where(q[..., :1] < 0, -q, q).to(DEV)
    from oracle import structure_oracle as SO
    rot = SO.quaternion_to_matrix(q.double()).float().contiguous()
    trans = (torch.randn(1, n, 3, generator=g) * 3).to(DEV)
    mask = _mask(n, "padded") if n > 1 else None
    return single, pair, q, trans, rot, mask


def _run_layers(pk, single, pair, quat, trans, rot, mask, shards=None, depth=2):
    """depth layers of the whole entry (shards None) or of begin per shard + concatenation + end; returns every per-residue
    tensor they write."""
    from alphafold2_b200 import ops
    s, q, t, r = single.clone(), quat.clone(), trans.clone(), rot.clone()
    n = s.shape[1]
    coords, conf = torch.full((1, n, 3), float("nan"), device=DEV), torch.full((1, n, 1), float("nan"), device=DEV)
    for i in range(depth):
        last = i == depth - 1
        c, f = (coords, conf) if last else (None, None)
        if shards is None:
            ops.structure_layer_(pk, s, pair, mask, q, t, r, c, f)
            continue
        o = torch.cat([ops.structure_layer_rows_begin_(pk, s, pair[:, a:b].contiguous(), mask, q, t, r, a)
                       for a, b in zip(shards, shards[1:])], 1)
        ops.structure_layer_rows_end_(pk, s, o, q, t, r, c, f)
    return {"single": s, "quat": q, "trans": t, "rot": r, "coords": coords, "confidence": conf}


@pytest.mark.parametrize("d", [32, 128])
@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("n", [1, 37])
def test_structure_layer_begin_end_whole_bitwise(n, H, d):
    model = _layer_model(d, H, seed=n + H + d)
    pk = model.structure_weights().packed()
    args = _layer_inputs(n, d, seed=n * 7 + H)
    want = _run_layers(pk, *args)
    got = _run_layers(pk, *args, shards=[0, n])
    assert torch.isfinite(want["coords"]).all()
    for k in want:
        assert _same(got[k], want[k]), k


@pytest.mark.parametrize("P", [2, 3, 4, 8])
def test_structure_layer_row_shards_bitwise(P):
    from alphafold2_b200 import parallel
    n, d, H = 37, 64, 4                                    # 37 rows: uneven shards at every P
    model = _layer_model(d, H, seed=P)
    pk = model.structure_weights().packed()
    args = _layer_inputs(n, d, seed=100 + P)
    want = _run_layers(pk, *args)
    got = _run_layers(pk, *args, shards=parallel.shard_offsets(n, P))
    for k in want:
        assert _same(got[k], want[k]), (P, k)


@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_pair_projection_rows_bitwise(precision):
    import alphafold2_b200 as A
    ops = _ops()
    n, d = 45, 64
    model = A.set_precision(_layer_model(d, 1, seed=3), precision)
    pk = model.pair_projection().packed()
    x = torch.randn(1, n, n, d, device=DEV)
    whole = ops.pair_projection_(pk, x.clone())
    for row0, rows in ((0, n), (0, 12), (13, 11), (n - 5, 5)):
        for band in (None, 1, 4):
            got = ops.pair_projection_rows_(pk, x[:, row0:row0 + rows].clone(), band=band)
            assert _same(got, whole[:, row0:row0 + rows]), (row0, rows, band)


def _rejected(fn, args, outs, code=BAD_ARG):
    lib = _lib()
    for o in outs:
        o.fill_(float("nan"))
    torch.cuda.synchronize()
    n0 = lib.af2_launch_count()
    rc = getattr(lib, fn)(*args, _ops()._stream_ptr())
    torch.cuda.synchronize()
    assert rc == code, (fn, args, rc)
    assert lib.af2_launch_count() == n0, f"{fn}: a rejected call launched a kernel"
    for o in outs:
        assert torch.isnan(o).all(), f"{fn}: a rejected call wrote its output"


def test_rows_entries_reject_malformed_calls():
    import ctypes as C
    ops = _ops()
    n, d, H, row0, rows = 20, 32, 2, 4, 6
    f = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    P = lambda t: t.data_ptr()  # noqa: E731
    proj, pair = f(n, 84 * H + 4), f(rows * n * d + 4)
    wb, bb, pw, R, t = f(H, d), f(H), f(H), f(n, 9), f(n, 3)
    out = f(rows, H * (32 + d))
    ok = [P(proj), P(pair), P(wb), P(bb), P(pw), None, P(R), P(t), P(out), n, row0, rows, H, d]

    def bad(**kw):
        a = list(ok)
        names = ["proj", "pair", "wb", "bb", "pw", "mask", "R", "t", "out", "n", "row0", "rows", "H", "d"]
        for k, v in kw.items():
            a[names.index(k)] = v
        return a

    for args in [bad(proj=None), bad(pair=None), bad(wb=None), bad(bb=None), bad(pw=None), bad(R=None), bad(t=None),
                 bad(out=None), bad(pair=P(pair) + 4), bad(proj=P(proj) + 4), bad(row0=-1), bad(rows=0), bad(rows=-2),
                 bad(row0=n - rows + 1), bad(row0=n), bad(n=0), bad(H=0), bad(H=17), bad(d=30), bad(d=1028)]:
        _rejected("af2_ipa_attention_rows", args, [out])

    model = _layer_model(d, H, seed=0)
    pk = model.structure_weights().packed()
    lib = _lib()
    single, q, o_rows, o = f(n, d), f(n, 4), f(rows, d), f(n, d)
    coords, conf = f(n, 3), f(n, 1)
    ws = f(lib.af2_structure_layer_rows_workspace(n, rows, d, H) // 4 + 1)
    W = C.byref(pk.struct)
    begin = [W, P(single), P(pair), None, P(q), P(t), P(R), P(o_rows), n, row0, rows, d, H, P(ws), ws.numel() * 4]
    end = [W, P(single), P(o), P(q), P(t), P(R), P(coords), P(conf), n, d, H, 1e-5, P(ws), ws.numel() * 4]

    def edit(base, **kw):
        a = list(base)
        for k, v in kw.items():
            a[int(k[1:])] = v
        return a

    no_points = _lib_struct_without(pk, "w_points")
    for args in [edit(begin, a0=None), edit(begin, a1=None), edit(begin, a2=None), edit(begin, a4=None), edit(begin, a5=None),
                 edit(begin, a6=None), edit(begin, a7=None), edit(begin, a13=None), edit(begin, a2=P(pair) + 4),
                 edit(begin, a9=-1), edit(begin, a10=0), edit(begin, a9=n - rows + 1), edit(begin, a8=0), edit(begin, a12=17),
                 edit(begin, a11=30), edit(begin, a0=C.byref(_lib_struct_without(pk, "w_proj")))]:
        _rejected("af2_structure_layer_rows_begin", args, [o_rows])
    _rejected("af2_structure_layer_rows_begin", edit(begin, a14=1024), [o_rows], code=WORKSPACE)
    for args in [edit(end, a0=None), edit(end, a1=None), edit(end, a2=None), edit(end, a3=None), edit(end, a4=None),
                 edit(end, a5=None), edit(end, a12=None), edit(end, a7=None), edit(end, a8=0), edit(end, a10=17),
                 edit(end, a9=30), edit(end, a0=C.byref(no_points)), edit(end, a0=C.byref(_lib_struct_without(pk, "w_qu")))]:
        _rejected("af2_structure_layer_rows_end", args, [single, coords, conf])
    _rejected("af2_structure_layer_rows_end", edit(end, a13=1024), [single, coords, conf], code=WORKSPACE)

    # the host wrappers check shapes before any call
    sg, pr = torch.randn(1, n, d, device=DEV), torch.randn(1, rows, n, d, device=DEV)
    q1, t1, R1 = q.view(1, n, 4), t.view(1, n, 3), R.view(1, n, 3, 3)
    with pytest.raises(ValueError, match="not inside"):
        ops.structure_layer_rows_begin_(pk, sg, pr, None, q1, t1, R1, n - rows + 1)
    with pytest.raises(ValueError, match="pair_rows"):
        ops.structure_layer_rows_begin_(pk, sg, pr[..., :16].contiguous(), None, q1, t1, R1, 0)
    with pytest.raises(ValueError, match="single and o"):
        ops.structure_layer_rows_end_(pk, sg, torch.randn(1, rows, d, device=DEV), q1, t1, R1)
    with pytest.raises(ValueError, match="not inside"):
        ops.ipa_attention_rows(proj[:, :84 * H].contiguous()[None], pr, wb, bb, pw, None, R1, t1, H, -1)
    with pytest.raises(ValueError, match="projection square"):
        ops.pair_projection_rows_(model.pair_projection().packed(), torch.randn(rows, n, d, device=DEV))


def _lib_struct_without(pk, field):
    """A copy of the packed af2_structure_weights with one pointer null."""
    from alphafold2_b200 import _lib as L
    s = L.StructureWeights(*(getattr(pk.struct, k) for k, _ in L.StructureWeights._fields_))
    setattr(s, field, None)
    return s
