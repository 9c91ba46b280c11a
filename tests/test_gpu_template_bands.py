"""-m gpu: the pointwise template attention in bands of pair rows (ops.TemplateAttentionRows through
Alphafold2.embed_templates_, and af2_template_pointwise_rows_begin / _group / _end).

q, gate and k|v are GEMM rows, the carry kernel resumes the softmax state exactly and to_out works row by row, so every band
computes each element from the same bits in the same order as the whole-tensor calls: bitwise equality, never a tolerance.
  * model: embed_templates_ with forced bands of 8, 16 and 64 rows and G in {1, 2, T} == band None, G = T, over batch, T, n
    (136: a ragged last band) and the "mixed" masks of test_gpu_template_groups.py; Alphafold2.forward on the
    alphafold2_templates.pt inputs with bands of 8;
  * C ABI: the rows entry points on a window inside larger tensors == the whole-tensor call on those rows, NaN guards around
    the window's outputs and state untouched; bad arguments return AF2_ERR_BAD_ARG and launch nothing;
  * memory: at N_res 1024, 4 templates, bands of 256 rows lower the peak below the one-template-at-a-time peak by at least
    what template_branch_bytes computes, and stay within the planned bytes;
  * long proteins (skipped without the free memory): N_res 2048 with bands of 512 == one template at a time; N_res 3072 with
    4 templates, which only fits in bands, runs and gives a finite, symmetric distogram.
"""
import functools

import pytest
import torch

from oracle import evoformer_oracle as O
from test_gpu_template_groups import _inputs, _model
from test_gpu_templates import _af2, _templates_fixture

pytestmark = pytest.mark.gpu

GB = 10 ** 9
AF2_ERR_BAD_ARG = -1


def _bits(t):
    return t.contiguous().view(torch.int32)


def _embed(model, x, x_mask, feats, tm, group, band):
    out = x.clone()
    with torch.no_grad():
        model.embed_templates_(out, x_mask, feats, tm, group=group, band=band)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------------------------------
# model: embed_templates_
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masks", ["ones", "mixed"])
@pytest.mark.parametrize("n", [24, 40, 136])
@pytest.mark.parametrize("T", [1, 3, 5])
@pytest.mark.parametrize("b", [1, 2])
def test_embed_templates_bands_bitwise(b, T, n, masks):
    model = _model("bf16")
    x, x_mask, feats, tm = _inputs(b, T, n, masks, seed=b * 1000 + T * 100 + n + 7)
    ref = _embed(model, x, x_mask, feats, tm, T, None)
    assert model.last_template_band == n and model.last_template_group == T
    assert not torch.equal(ref, x), "the template branch changed nothing: the test would prove nothing"
    for band in (8, 16, 64):
        if band >= n:
            continue
        for G in sorted({1, 2, T}):
            if G > T:
                continue
            out = _embed(model, x, x_mask, feats, tm, G, band)
            assert model.last_template_band == band and model.last_template_group == G
            assert torch.equal(_bits(out), _bits(ref)), \
                f"b{b} T{T} n{n} {masks}: bands of {band}, G = {G} differ (max |diff| {(out - ref).abs().max().item():.3e})"


def test_forced_band_must_be_a_multiple_of_8():
    model = _model("bf16")
    x, x_mask, feats, tm = _inputs(1, 2, 40, "ones", seed=3)
    x0 = x.clone()
    for band in (12, 0, -8):
        with pytest.raises(ValueError, match="multiple of 8"):
            model.embed_templates_(x, x_mask, feats, tm, band=band)
    assert torch.equal(x, x0)


def test_strict_mode_ignores_the_band():
    model = _model("strict")
    x, x_mask, feats, tm = _inputs(1, 3, 40, "mixed", seed=4)
    ref = _embed(model, x, x_mask, feats, tm, 3, None)
    out = _embed(model, x, x_mask, feats, tm, 1, 8)
    assert model.last_template_band == 40
    assert torch.equal(_bits(out), _bits(ref))


def test_alphafold2_templates_fixture_bands_of_8_bitwise():
    fx = _templates_fixture()
    i = {k: v.cuda() for k, v in fx["inputs"].items()}
    model = _af2(fx["cfg"], fx["state"], "bf16")
    kw = {k: i[k] for k in fx["calls"]["feats_angles"]}
    with torch.no_grad():
        ref = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], **kw).distance
        n = i["seq"].shape[1]
        assert model.last_template_band == n and n > 8
        model.embed_templates_ = functools.partial(type(model).embed_templates_, model, band=8)
        out = model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], **kw).distance
    torch.cuda.synchronize()
    assert model.last_template_band == 8
    assert torch.equal(_bits(out), _bits(ref)), f"max |diff| {(out - ref).abs().max().item():.3e}"


# ------------------------------------------------------------------------------------------------------------------------
# C ABI: the rows entry points
# ------------------------------------------------------------------------------------------------------------------------
def _attn_weights(d, heads, dh, seed):
    from alphafold2_b200 import ops
    g = torch.Generator().manual_seed(seed)
    I = heads * dh
    w = [torch.randn(I, d, generator=g) * d ** -0.5, torch.randn(2 * I, d, generator=g) * d ** -0.5,
         torch.randn(I, d, generator=g) * d ** -0.5, torch.randn(I, generator=g), torch.randn(d, I, generator=g) * I ** -0.5,
         torch.randn(d, generator=g)]
    return ops.pack_template_attention(*(t.cuda() for t in w), dh)


GUARD = 4096          # elements of NaN before and after every window buffer (a multiple of 16 bytes for each dtype)


def _guarded(rows, cols, dtype):
    buf = torch.full((rows * cols + 2 * GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + rows * cols]


@pytest.mark.parametrize("groups", [(1,), (2,), (3,), (1, 2), (2, 1), (1, 1, 1)])
def test_rows_entry_points_on_a_window(groups):
    import ctypes as C
    from alphafold2_b200 import _lib, ops
    lib = _lib.load()
    B, n, d, heads, dh = 2, 40, 64, 2, 32
    T, I, nn = sum(groups), heads * dh, n * n
    pk = _attn_weights(d, heads, dh, seed=len(groups) * 10 + T)
    g = torch.Generator().manual_seed(T + 100 * len(groups))
    x = torch.randn(B, n, n, d, generator=g).cuda()
    t = torch.randn(B, T, n, n, d, generator=g).cuda()
    xm = (torch.rand(B, n, n, generator=g) > 0.15).cuda()
    tm = torch.rand(B, T, n, n, generator=g) > 0.3
    tm[:, :, 10:13] = False                                # pairs with every template masked
    tm[1 if T > 1 else 0, 0] = False                       # a fully masked template (in the window's batch element if T > 1)
    tm = tm.cuda()
    ref = x.clone()
    ops.template_pointwise_attention_(pk, ref, t.reshape(B * T, n, n, d), xm, tm.reshape(B * T, n, n), heads, dh)
    # window: batch element 1, pair rows [8, 24)
    b, i0, i1 = 1, 8, 24
    P, o = (i1 - i0) * n, b * nn + i0 * n
    xw = x.clone()
    st = {k: _guarded(B * nn, c, torch.float32) for k, c in (("run_max", heads), ("run_sum", heads), ("acc", I), ("pooled", 1))}
    win = {k: (buf, ops._addr(buf, GUARD + o * c)) for (k, (buf, _)), c in zip(st.items(), (heads, heads, I, 1))}
    qb, q = _guarded(P, I, torch.bfloat16)
    gb, gate = _guarded(P, I, torch.bfloat16)
    s = ops._stream_ptr()
    w = C.byref(pk.struct)
    ws = ops.workspace(max(lib.af2_template_pointwise_rows_begin_workspace(P, d),
                           lib.af2_template_pointwise_rows_group_workspace(max(groups), P, d, heads, dh)), "cuda")
    t0 = 0
    for k, G in enumerate(groups):
        first, last = int(k == 0), int(k == len(groups) - 1)
        _lib.check(lib.af2_template_pointwise_rows_begin(w, ops._addr(xw, o * d), P, d, heads, dh, q.data_ptr(), gate.data_ptr(),
                                                         ws.data_ptr(), ws.numel(), s))
        # template g of the group: t[b, t0 + g], i.e. a stride of n^2 pairs inside t [B, T, n, n, d]
        base = (b * T + t0) * nn + i0 * n
        _lib.check(lib.af2_template_pointwise_rows_group(
            w, ops._addr(t, base * d), ops._addr(xm, o), ops._addr(tm, base), G, P, nn, d, heads, dh, q.data_ptr(), gate.data_ptr(),
            win["run_max"][1], win["run_sum"][1], win["acc"][1], win["pooled"][1], q.data_ptr(), first, last, ws.data_ptr(),
            ws.numel(), s))
        t0 += G
    _lib.check(lib.af2_template_pointwise_rows_end(w, ops._addr(xw, o * d), q.data_ptr(), win["pooled"][1], P, d, heads, dh,
                                                   ws.data_ptr(), 0, s))
    torch.cuda.synchronize()
    flat, rflat, x0 = xw.view(-1, d), ref.view(-1, d), x.view(-1, d)
    assert torch.equal(_bits(flat[o:o + P]), _bits(rflat[o:o + P])), \
        f"{groups}: window differs from the whole call (max |diff| {(flat[o:o + P] - rflat[o:o + P]).abs().max().item():.3e})"
    assert not torch.equal(flat[o:o + P], x0[o:o + P])
    assert torch.equal(_bits(flat[:o]), _bits(x0[:o])) and torch.equal(_bits(flat[o + P:]), _bits(x0[o + P:])), \
        "rows outside the window changed"
    for buf in (qb, gb):
        assert buf[:GUARD].isnan().all() and buf[-GUARD:].isnan().all(), "a write outside q / gate"
    for name, (buf, _), c in zip(st, st.values(), (heads, heads, I, 1)):
        lo, hi = GUARD + o * c, GUARD + (o + P) * c
        assert buf[:lo].isnan().all() and buf[hi:].isnan().all(), f"a write outside the window's {name}"
    pooled = st["pooled"][1][o:o + P]
    assert pooled.isfinite().all() and pooled.eq(tm[b].reshape(T, -1)[:, i0 * n:i1 * n].any(0).float()).all()


def test_rows_entry_points_reject_bad_arguments():
    import ctypes as C
    from alphafold2_b200 import _lib, ops
    lib = _lib.load()
    n, d, heads, dh = 16, 64, 2, 32
    I, P = heads * dh, 4 * n
    pk = _attn_weights(d, heads, dh, seed=5)
    x = torch.randn(1, n, n, d, device="cuda")
    t = torch.randn(2, n, n, d, device="cuda")
    x0 = x.clone()
    q = torch.full((P + 8, I), float("nan"), dtype=torch.bfloat16, device="cuda")
    gate = torch.full((P, I), float("nan"), dtype=torch.bfloat16, device="cuda")
    state = [torch.full((n * n, c), float("nan"), device="cuda") for c in (heads, heads, I, 1)]
    sp = [s.data_ptr() for s in state]
    ws = ops.workspace(lib.af2_template_pointwise_rows_group_workspace(2, P, d, heads, dh), "cuda")
    s = ops._stream_ptr()
    w = C.byref(pk.struct)
    wsa = (ws.data_ptr(), ws.numel(), s)

    def begin(w=w, x=x.data_ptr(), P=P, q=q.data_ptr()):
        return lib.af2_template_pointwise_rows_begin(w, x, P, d, heads, dh, q, gate.data_ptr(), *wsa)

    def group(w=w, t=t.data_ptr(), G=2, P=P, stride=n * n, q=q.data_ptr(), st=sp, first=0, last=0):
        return lib.af2_template_pointwise_rows_group(w, t, None, None, G, P, stride, d, heads, dh, q, gate.data_ptr(), *st,
                                                     q, first, last, *wsa)

    def end(w=w, x=x.data_ptr(), P=P, out=q.data_ptr(), pooled=sp[3]):
        return lib.af2_template_pointwise_rows_end(w, x, out, pooled, P, d, heads, dh, *wsa)

    bad = {
        "begin null weights": begin(w=None), "begin null x": begin(x=None), "begin negative P": begin(P=-1),
        "begin misaligned x": begin(x=x.data_ptr() + 4), "begin misaligned q": begin(q=q.data_ptr() + 2),
        "group null weights": group(w=None), "group null t": group(t=None), "group negative P": group(P=-n),
        "group misaligned t": group(t=t.data_ptr() + 4), "group misaligned q": group(q=q.data_ptr() + 2),
        "group first = 2": group(first=2), "group last = -1": group(last=-1), "group G = 0": group(G=0),
        "group stride below the window": group(stride=P - 1), "group null state": group(st=[None, None, None, sp[3]]),
        "group null pooled": group(st=sp[:3] + [None]), "group misaligned acc": group(st=sp[:2] + [sp[2] + 4, sp[3]]),
        "end null weights": end(w=None), "end null x": end(x=None), "end negative P": end(P=-1),
        "end misaligned out": end(out=q.data_ptr() + 2), "end null pooled": end(pooled=None),
    }
    torch.cuda.synchronize()
    wrong = {k: rc for k, rc in bad.items() if rc != AF2_ERR_BAD_ARG}
    assert not wrong, f"expected AF2_ERR_BAD_ARG ({AF2_ERR_BAD_ARG}): {wrong}"
    assert q.isnan().all() and gate.isnan().all() and all(s.isnan().all() for s in state), "a rejected call launched work"
    assert torch.equal(x, x0)
    # P = 0 is a valid empty window
    assert begin(P=0) == 0 and group(P=0) == 0 and end(P=0) == 0


# ------------------------------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _big_model(layers=2):
    import alphafold2_b200 as A
    torch.manual_seed(8)
    model = A.Alphafold2(dim=256, depth=1, heads=8, dim_head=64, templates_dim=32, templates_embed_layers=layers, max_seq_len=4096)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    return model.cuda().eval()


def _peak(model, x, x_mask, feats, tm, group, band):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        model.embed_templates_(x, x_mask, feats, tm, group=group, band=band)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ops._WORKSPACE.clear()
    return peak


def test_bands_lower_the_peak_by_what_the_planner_computes():
    from alphafold2_b200 import ops
    n, T, d = 1024, 4, 256
    model = _big_model()
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(1, n, n, d, device="cuda", generator=g)
    x_mask = torch.ones(1, n, n, dtype=torch.bool, device="cuda")
    feats = torch.randn(1, T, n, n, 32, device="cuda", generator=g)
    tm = torch.ones(1, T, n, dtype=torch.bool, device="cuda")
    one = _peak(model, x.clone(), x_mask, feats, tm, 1, None)
    assert model.last_template_band == n
    banded = _peak(model, x.clone(), x_mask, feats, tm, 1, 256)
    assert model.last_template_band == 256
    plan_one = ops.template_branch_bytes(1, T, 1, n, d, 8, 64, "bf16", 32)
    plan_band = ops.template_branch_bytes(1, T, 1, n, d, 8, 64, "bf16", 32, band=256)
    print(f"N {n} T {T}: peak one template at a time {one / GB:.3f} GB, bands of 256 {banded / GB:.3f} GB; planned "
          f"{plan_one / GB:.3f} / {plan_band / GB:.3f} GB")
    assert one - banded >= plan_one - plan_band, f"saved {(one - banded) / GB:.3f} GB, planned {(plan_one - plan_band) / GB:.3f} GB"
    assert banded <= plan_band, "the planner under-counts the banded branch"


# ------------------------------------------------------------------------------------------------------------------------
# long proteins
# ------------------------------------------------------------------------------------------------------------------------
def _need(gb):
    from alphafold2_b200 import ops
    ops._WORKSPACE.clear()
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip(f"needs {gb} GB free on the device, {free / GB:.1f} GB of {total / GB:.1f} GB are")


def _long_inputs(n, T, S=8, seed=10):
    g = torch.Generator(device="cuda").manual_seed(seed)
    seq = torch.randint(0, 21, (1, n), device="cuda", generator=g)
    msa = torch.randint(0, 21, (1, S, n), device="cuda", generator=g)
    mask = torch.ones(1, n, dtype=torch.bool, device="cuda")
    mask[:, -5:] = False
    feats = torch.randn(1, T, n, n, 32, device="cuda", generator=g)
    tm = torch.rand(1, T, n, device="cuda", generator=g) > 0.1
    return dict(seq=seq, msa=msa, mask=mask, msa_mask=torch.ones(1, S, n, dtype=torch.bool, device="cuda"), templates_feats=feats,
                templates_mask=tm)


def _forward(model, i, **kw):
    model.embed_templates_ = functools.partial(type(model).embed_templates_, model, **kw)
    try:
        with torch.no_grad():
            return model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"], templates_feats=i["templates_feats"],
                         templates_mask=i["templates_mask"]).distance
    finally:
        del model.embed_templates_


def test_n2048_bands_of_512_equal_one_template_at_a_time():
    _need(70)
    n, T = 2048, 4
    model = _big_model(layers=1)
    i = _long_inputs(n, T)
    ref = _forward(model, i, group=1)
    assert model.last_template_band == n
    out = _forward(model, i, group=1, band=512)
    torch.cuda.synchronize()
    assert model.last_template_band == 512
    assert torch.equal(_bits(out), _bits(ref)), f"max |diff| {(out - ref).abs().max().item():.3e}"


def test_n3072_four_templates_run_in_bands():
    _need(75)
    n, T = 3072, 4
    model = _big_model(layers=1)
    i = _long_inputs(n, T, seed=11)
    # a forward without templates first: it leaves the grow-only workspace at the trunk's size, which the banded branch
    # counts as free and must release before it allocates the softmax state
    with torch.no_grad():
        model(i["seq"], i["msa"], mask=i["mask"], msa_mask=i["msa_mask"])
    torch.cuda.reset_peak_memory_stats()
    dist = _forward(model, i)
    torch.cuda.synchronize()
    print(f"N {n} T {T}: template bands of {model.last_template_band} rows, G {model.last_template_group}, "
          f"peak {torch.cuda.max_memory_allocated() / GB:.1f} GB")
    assert model.last_template_band < n
    assert bool(torch.isfinite(dist).all())
    assert torch.equal(_bits(dist), _bits(dist.transpose(1, 2)))
