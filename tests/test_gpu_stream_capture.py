"""-m gpu: the promise of INTEGRATION.md §C, entry point by entry point: launches are asynchronous on the caller's stream and
CUDA-graph capturable.  Every scenario runs its op in two modes:
  (a) caller's stream: on a side stream, a ~10^8-cycle sleep, the inputs written there with copy_, then the op there; the
      output must be bitwise a default-stream run's.  A launch, memset or copy issued on another stream reads the inputs
      before they are written.
  (b) capture: warm up, capture with torch.cuda.graph on static inputs, fill the inputs with new values and replay; the
      output must be bitwise eager on those values.
Scenarios that cannot be captured (NOT_CAPTURABLE, with the reason) run in mode (a) only.
A recording wrapper around every af2_* symbol of the library notes which entries the scenarios reach; the last test asserts
that every entry issuing device work was reached or is listed in EXCLUDED with its reason, and that no EXCLUDED entry was
reached (a stale exclusion fails).
The workspace lifetime test captures an op, grows and releases the shared workspace, and checks that the buffer the graph
points into is still alive (ops.workspace retains it) before it replays."""
import gc
import weakref

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")]

DEV = torch.device("cuda", 0)
SLEEP_CYCLES = 100_000_000

# entries of _lib._SIGNATURES that launch nothing (besides every *_workspace size query): they may or may not be called
QUERY_ONLY = {"af2_last_error", "af2_abi_version", "af2_check_device", "af2_launch_count", "af2_profile_enable", "af2_profile_read",
              "af2_attention_proj_max_n", "af2_ipa_tile_rows", "af2_peer_ctrl_bytes", "af2_peer_can_access",
              "af2_chan_to_token_select"}
# entries that issue device work but that no scenario here reaches, with the reason; none of them may be called here
PEER = "peer-memory exchange of the sharded trunk: needs P >= 2 ranks with IPC-mapped arenas"
SHARDED = ("tied-query column attention over column shards: only the sharded schedule issues it (the one-GPU banded path "
           "refuses tied queries); replayed in the sharded trunk's graph by tests/test_gpu_graph_replay.py")
NO_CALLER = "no Python code of the package issues it: a kernel-level entry of the kernel-by-kernel tests"


def _wrapper(fn):
    return f"issued only by the kernel-level wrapper ops.{fn}, which no module, model or utils function calls (the kernel tests do)"


EXCLUDED = {
    **{k: PEER for k in ("af2_peer_alloc", "af2_peer_free", "af2_peer_export", "af2_peer_open", "af2_peer_close",
                         "af2_peer_error", "af2_peer_exchange", "af2_peer_exchange_chunks")},
    "af2_axial_attention_tied_begin": SHARDED, "af2_axial_attention_tied_end": SHARDED,
    "af2_attention_bf16": _wrapper("attention_bf16"), "af2_attention_proj_bf16": _wrapper("attention_proj_bf16"),
    "af2_chan_to_token": _wrapper("chan_to_token"), "af2_contract_tail": _wrapper("contract_tail"),
    "af2_gemm_bf16_epilogue": _wrapper("gemm_bf16_epilogue"), "af2_gemm_bf16_f32": _wrapper("gemm_bf16"),
    "af2_gemm_bf16_f32_gathered": _wrapper("gemm_bf16_f32_strided"), "af2_gemm_split_f32": _wrapper("gemm_split"),
    "af2_split_bf16": _wrapper("gemm_split"), "af2_ipa_attention_rows": _wrapper("ipa_attention_rows"),
    "af2_layernorm_bf16": _wrapper("layernorm_bf16"), "af2_outer_scale": _wrapper("outer_scale"),
    "af2_template_pointwise_bf16_state": _wrapper("template_pointwise"), "af2_template_pointwise_f32_state": _wrapper("template_pointwise"),
    **{k: NO_CALLER for k in ("af2_axial_attention", "af2_gemm_split_epilogue", "af2_strict_ln_split", "af2_strict_geglu_split",
                              "af2_strict_gelu_split", "af2_strict_qkv_split", "af2_strict_pair_bias", "af2_strict_softmax_split",
                              "af2_strict_gate_split", "af2_strict_tok2chan_split", "af2_strict_chan_to_token", "af2_tie_queries_f32",
                              "af2_tie_queries_bf16", "af2_attention_x_bf16", "af2_attn_bias_log2", "af2_strict_xqkv_split",
                              "af2_strict_xsoftmax_split", "af2_strict_xgate_split")},
}


# ------------------------------------------------------------------------------------------------------------
# coverage recorder
# ------------------------------------------------------------------------------------------------------------
CALLED = set()
RAN = set()


@pytest.fixture(scope="module", autouse=True)
def _record_calls():
    from alphafold2_b200 import _lib
    lib = _lib.load()
    orig = {name: getattr(lib, name) for name in _lib._SIGNATURES}
    for name, fn in orig.items():
        def rec(*a, _fn=fn, _name=name):
            CALLED.add(_name)
            return _fn(*a)
        setattr(lib, name, rec)
    yield
    for name, fn in orig.items():
        setattr(lib, name, fn)


# ------------------------------------------------------------------------------------------------------------
# the two modes
# ------------------------------------------------------------------------------------------------------------
def _tensors(o):
    if torch.is_tensor(o):
        return [o]
    if isinstance(o, (tuple, list)):
        return [t for x in o for t in _tensors(x)]
    if hasattr(o, "__dict__"):
        return [t for k in sorted(vars(o)) for t in _tensors(vars(o)[k])]
    return []


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8) if t.dtype != torch.bool else t


def _assert_same(got, want, what):
    got, want = _tensors(got), _tensors(want)
    assert len(got) == len(want) and len(want) > 0, (what, len(got), len(want))
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if a.shape != b.shape or a.dtype != b.dtype or
           not torch.equal(_bits(a), _bits(b))]
    assert not bad, f"{what}: outputs {bad} of {len(want)} differ"


def _dev(kw):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in kw.items()}


def _caller_stream(fn, kw, name):
    src = _dev(kw)
    want = _tensors(fn(**{k: (v.clone() if torch.is_tensor(v) else v) for k, v in src.items()}))
    want = [t.clone() for t in want]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        ins = {k: (torch.empty_like(v).copy_(v) if torch.is_tensor(v) else v) for k, v in src.items()}
        got = _tensors(fn(**ins))
    torch.cuda.synchronize()
    _assert_same(got, want, f"{name}: on the caller's stream")


def _capture(fn, kw, kw_new, name):
    from alphafold2_b200 import ops
    static = _dev(kw)
    cur = torch.cuda.current_stream()
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        fn(**static)
    cur.wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn(**static)
    new = _dev(kw_new)
    for k, v in new.items():
        if torch.is_tensor(v):
            static[k].copy_(v)
    g.replay()
    torch.cuda.synchronize()
    want = fn(**{k: (v.clone() if torch.is_tensor(v) else v) for k, v in new.items()})
    torch.cuda.synchronize()
    _assert_same(out, want, f"{name}: graph replay on new inputs")
    del g, out
    gc.collect()
    ops.release_captured_workspaces()


# ------------------------------------------------------------------------------------------------------------
# scenarios: name -> () -> (fn, inputs(seed) -> dict of CPU tensors and plain values)
# ------------------------------------------------------------------------------------------------------------
def _init(module, seed=0):
    from oracle import evoformer_oracle as O
    module.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in module.state_dict().items()}, std=0.05, seed=seed))
    return module.to(DEV).eval()


def _evoformer_module(precision, tied=False):
    """An Evoformer of depth 2 (d 64, N_res 40, S 6) and its masked inputs(seed)."""
    import alphafold2_b200 as A
    torch.manual_seed(0)
    d, N, S = 64, 40, 6
    evo = A.set_precision(_init(A.Evoformer(depth=2, dim=d, seq_len=N, heads=2, dim_head=32, attn_dropout=0., ff_dropout=0.,
                                            global_column_attn=tied)), precision)

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        m1 = torch.rand(1, N, generator=g) > 0.15
        m1[:, 0] = True
        msa_mask = torch.rand(1, S, N, generator=g) > 0.1
        msa_mask[:, 0] = True
        return dict(x=torch.randn(1, N, N, d, generator=g), m=torch.randn(1, S, N, d, generator=g),
                    mask=m1[:, :, None] & m1[:, None, :], msa_mask=msa_mask)
    return evo, inputs


def _evoformer(precision, tied=False):
    evo, inputs = _evoformer_module(precision, tied)
    return lambda x, m, mask, msa_mask: evo(x, m, mask=mask, msa_mask=msa_mask), inputs


def _attention(strict):
    import test_gpu_attention_forward as AF
    d, heads = 64, 4
    a, _ = AF._module(d, heads, 12 if strict else 32, strict=strict, seed=7)

    def inputs(seed):
        kw = AF._inputs(6, 40, 23, d, heads, seed=seed, bias="1hij")
        kw["tie_dim"] = 3
        return kw
    return lambda **kw: a(**kw), inputs


def _model(n=24, **kw):
    import test_gpu_recycle_loop as RL
    return RL._model(d=128, depth=1, sdepth=1, n=n, predict_angles=True, **kw)


def _templates(group, band, precision="bf16"):
    model = _model(precision=precision)
    n, T, d = 24, 3, 128

    def run(x, x_mask, feats, tmask):
        y = x.clone()
        model.embed_templates_(y, x_mask, feats, tmask, group=group, band=band)
        return y

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        m1 = torch.rand(1, n, generator=g) > 0.15
        tmask = torch.rand(1, T, n, generator=g) > 0.1
        return dict(x=torch.randn(1, n, n, d, generator=g), x_mask=m1[:, :, None] & m1[:, None, :],
                    feats=torch.randn(1, T, n, n, 32, generator=g), tmask=tmask)
    return run, inputs


def _glue(precision="bf16"):
    """Pair init (whole and rows), the recycling embedder (whole and rows), the template angle rows, the distogram and angle
    heads (whole and rows)."""
    import alphafold2_b200 as A
    from alphafold2_b200 import ops
    model = _model(precision=precision)
    n, S, T, d, r0, r1 = 24, 3, 2, 128, 8, 20
    ln, lin = model.to_distogram_logits[0], model.to_distogram_logits[1]
    emb = (model.token_emb.weight, model.to_pairwise_repr.weight, model.to_pairwise_repr.bias, model.pos_emb.weight, model.max_rel_dist)

    def run(seq, msa, msa_mask, coords, single, pair, angles, tmask):
        rec = A.Recyclables(coords, single, pair)
        x, m = ops.embed_pair_init(seq, msa, *emb, m_rows=S + T)
        model.embed_recyclables_(x, m, rec)
        mm = model.embed_template_angles_(m, msa_mask, angles, tmask)
        xr, mr = ops.embed_pair_init_rows(seq, msa, *emb, r0, r1 - r0, m_rows=S)
        model.embed_recyclables_(xr, mr, rec, row0=r0)
        heads = model.angle_heads()
        rows, cols = x[0, r0:r1].contiguous(), x[0, :, r0:r1].contiguous()
        return (x, m, mm, xr, mr, ops.distogram_head(x, ln.weight, ln.bias, lin.weight, lin.bias), heads.run(x, True),
                ops.distogram_head_rows(rows, cols, ln.weight, ln.bias, lin.weight, lin.bias),
                ops.angle_heads_rows(heads.packed(), rows, cols, True))

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        return dict(seq=torch.randint(0, 21, (1, n), generator=g), msa=torch.randint(0, 21, (1, S, n), generator=g),
                    msa_mask=torch.rand(1, S, n, generator=g) > 0.1, coords=torch.randn(1, n, 3, generator=g) * 5,
                    single=torch.randn(1, n, d, generator=g), pair=torch.randn(1, n, n, d, generator=g),
                    angles=torch.randn(1, T, n, 55, generator=g), tmask=torch.rand(1, T, n, generator=g) > 0.1)
    return run, inputs


def _structure():
    """One structure layer (whole, then as the rows halves), with msa_to_single_repr_dim and the pair projection."""
    from alphafold2_b200 import ops
    from alphafold2_b200.alphafold2 import ReturnValues, structure_frames
    model = _model()
    n, d = 24, 128

    def run(x, m, mask):
        coords, ret = model._structure_module(x, m, mask, ReturnValues(), x_private=False, return_confidence=False,
                                              return_recyclables=True, return_aux_logits=True)
        pk = model.structure_weights().packed()
        single = ops.structure_linear(m[:, 0].contiguous(), model.msa_to_single_repr_dim.weight, model.msa_to_single_repr_dim.bias)
        pair = ops.pair_projection_rows_(model.pair_projection().packed(), x[:, 4:20].clone())
        quat, trans, rot, c2, conf2 = structure_frames(1, n, DEV)
        o = ops.structure_layer_rows_begin_(pk, single, pair, mask, quat, trans, rot, 4)
        o_all = torch.zeros(1, n, d, device=DEV)
        o_all[:, 4:20] = o
        ops.structure_layer_rows_end_(pk, single, o_all, quat, trans, rot, c2, conf2)
        return coords, ret.recyclables, c2, conf2, quat, trans

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        mask = torch.rand(1, n, generator=g) > 0.15
        return dict(x=torch.randn(1, n, n, d, generator=g), m=torch.randn(1, 3, n, d, generator=g), mask=mask)
    return run, inputs


def _evoformer_bands(band, msa_band):
    """The one-GPU Evoformer in bands of pair rows and MSA rows (banded.py through CudaStageOps), the path the planner takes
    for long proteins and deep MSAs; forced here at a small size."""
    evo, inputs = _evoformer_module("bf16")

    def run(x, m, mask, msa_mask):
        xo, mo = x.clone(), m.clone()
        evo.run_(xo, mo, mask, msa_mask, band=band, msa_band=msa_band)
        assert (evo.last_pair_band, evo.last_msa_band) == (min(band, x.shape[1]), msa_band)
        return xo, mo
    return run, inputs


def _rotary():
    import alphafold2_b200 as A
    b, h, n, dh, rot = 2, 4, 40, 32, 16

    def run(x, sin, cos):
        return A.apply_rotary_pos_emb(x, (sin, cos)), A.rotate_every_two(x)

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        return dict(x=torch.randn(b, h, n, dh, generator=g), sin=torch.randn(1, n, rot, generator=g), cos=torch.randn(1, n, rot, generator=g))
    return run, inputs


def _ipa_block():
    block = _model().ipa_block
    n, d = 24, 128

    def run(x, pair, rot, trans, mask):
        return block(x, pairwise_repr=pair, rotations=rot, translations=trans, mask=mask)

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        q, _ = torch.linalg.qr(torch.randn(1, n, 3, 3, generator=g))
        return dict(x=torch.randn(1, n, d, generator=g), pair=torch.randn(1, n, n, d, generator=g), rot=q,
                    trans=torch.randn(1, n, 3, generator=g) * 3, mask=torch.rand(1, n, generator=g) > 0.15)
    return run, inputs


def _mds():
    from alphafold2_b200 import ops
    n = 40

    def run(delta, weights, x0):
        x = x0.clone()
        steps, stopped, his, stress = ops.mds_iterate_(delta, weights, x, 6, 1e-5)
        return x, his, stress

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        pts = torch.randn(1, n, 3, generator=g) * 6
        return dict(delta=torch.cdist(pts, pts), weights=torch.rand(1, n, n, generator=g), x0=pts + torch.randn(1, n, 3, generator=g))
    return run, inputs


def _losses():
    from alphafold2_b200 import utils as U
    from test_gpu_angle_loss import backbone
    n = 40

    def run(dist_logits, coords, pred, mask, theta, phi, omega, bb):
        return (U.distogram_loss(dist_logits, coords, mask), U.angle_loss(theta, phi, omega, bb, mask),
                U.score_coords(pred, coords, mask), U.distmat_loss_torch(pred, coords), U.get_bucketed_distance_matrix(coords, mask),
                U.get_bucketed_angle_matrices(bb, mask))

    def inputs(seed):
        g = torch.Generator().manual_seed(seed)
        coords = torch.randn(1, n, 3, generator=g) * 8
        return dict(dist_logits=torch.randn(1, n, n, 37, generator=g), coords=coords,
                    pred=coords + torch.randn(1, n, 3, generator=g), mask=torch.rand(1, n, generator=g) > 0.15,
                    theta=torch.randn(1, n, n, 25, generator=g), phi=torch.randn(1, n, n, 13, generator=g),
                    omega=torch.randn(1, n, n, 25, generator=g), bb=backbone(1, n, g, 3, scale=4.0))
    return run, inputs


def _center_distogram():
    from alphafold2_b200 import utils as U
    return lambda distogram: U.center_distogram_torch(distogram), \
        lambda seed: dict(distogram=torch.softmax(torch.randn(1, 40, 40, 37, generator=torch.Generator().manual_seed(seed)), -1))


SCENARIOS = {
    "evoformer_bf16": lambda: _evoformer("bf16"),
    "evoformer_strict": lambda: _evoformer("strict"),
    "extra_msa_tied": lambda: _evoformer("bf16", tied=True),
    "extra_msa_tied_strict": lambda: _evoformer("strict", tied=True),
    "attention": lambda: _attention(False),
    "attention_strict": lambda: _attention(True),
    "templates_whole": lambda: _templates(None, None),
    "templates_groups": lambda: _templates(1, None),
    "templates_banded": lambda: _templates(None, 8),
    "templates_strict": lambda: _templates(None, None, "strict"),
    "templates_strict_groups": lambda: _templates(1, None, "strict"),
    "glue": lambda: _glue(),
    "glue_strict": lambda: _glue("strict"),
    "structure": _structure,
    "losses": _losses,
    "center_distogram": _center_distogram,
    "evoformer_pair_and_msa_bands": lambda: _evoformer_bands(16, 2),
    "evoformer_msa_bands": lambda: _evoformer_bands(40, 4),
    "rotary": _rotary,
    "ipa_block": _ipa_block,
    "mds_iterate": _mds,
}
# scenarios that run on the caller's stream but cannot be captured, with the reason (INTEGRATION.md §C lists them too)
NOT_CAPTURABLE = {
    "center_distogram": "the bin centres are computed from the CPU bins and copied to the device from pageable memory on every call",
    "mds_iterate": "ops.mds_iterate_ reads the step count back on the host after each call (the SMACOF loop's tolerance stop)",
}


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_caller_stream_and_capture(name):
    fn, inputs = SCENARIOS[name]()
    with torch.no_grad():
        _caller_stream(fn, inputs(1), name)
        if name not in NOT_CAPTURABLE:
            _capture(fn, inputs(1), inputs(2), name)
    RAN.add(name)


def test_captured_workspace_outlives_growth_and_release():
    """A graph that captured an op keeps its workspace buffer through a larger op and release_workspace()."""
    from alphafold2_b200 import ops
    fn, inputs = _evoformer("bf16")
    big, big_inputs = SCENARIOS["templates_whole"]()
    with torch.no_grad():
        ops.release_workspace(DEV)
        static = _dev(inputs(1))
        fn(**static)                                               # sizes the shared workspace
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn(**static)
        used = weakref.ref(ops._WORKSPACE[DEV])
        size = used().numel()
        big(**_dev(big_inputs(3)))                                 # grows the shared workspace
        torch.cuda.synchronize()
        assert ops._WORKSPACE[DEV].numel() > size
        ops.release_workspace(DEV)
        gc.collect()
        assert used() is not None, "the captured workspace was freed while the graph still points into it"
        junk = torch.full((1 << 28,), float("nan"), device=DEV)
        new = _dev(inputs(2))
        for k, v in new.items():
            static[k].copy_(v)
        g.replay()
        torch.cuda.synchronize()
        del junk
        _assert_same(out, fn(**new), "replay after the shared workspace grew and was released")
        del g, out
        ops.release_captured_workspaces()
        gc.collect()
        assert used() is None


def test_every_entry_is_reached():
    from alphafold2_b200 import _lib
    if RAN != set(SCENARIOS):
        pytest.skip(f"needs every scenario of this module in the same run; missing {sorted(set(SCENARIOS) - RAN)}")
    names = set(_lib._SIGNATURES)
    assert QUERY_ONLY <= names and set(EXCLUDED) <= names, sorted((QUERY_ONLY | set(EXCLUDED)) - names)
    stale = sorted(set(EXCLUDED) & CALLED)
    assert not stale, f"EXCLUDED lists entries the scenarios do reach: {stale}"
    device_work = {s for s in names if not s.endswith("_workspace")} - QUERY_ONLY - set(EXCLUDED)
    missing = sorted(device_work - CALLED)
    assert not missing, f"entries no scenario reached and EXCLUDED does not list: {missing}"
