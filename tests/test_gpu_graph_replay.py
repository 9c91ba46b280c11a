"""-m gpu: the CUDA-graph replay of the sharded trunk (parallel._GraphedTrunk), the default of shard_evoformer and
shard_alphafold2, on one GPU.  Each case runs in a spawned child process that holds a one-rank NCCL group (the collectives
are graph nodes) and releases its graphs before destroy_process_group.  Every case asserts that a graph was captured and
replayed (`_af2_graph.failed is None`), so none of them passes on the eager fallback.  Checks:
  * the trunk at the shapes of tests/test_gpu_parallel.py and one with S > N: the capturing call and a replay bitwise the
    eager schedule (use_graph=False) on the same inputs, and both against the fp64 oracle;
  * new inputs: new tensors, the held tensors changed in place, and a mask going from None to a tensor (a recapture);
  * weights: load_state_dict, p.copy_ and p.data.add_ + invalidate_packed each recapture and replay the new weights;
    set_precision("strict") refuses, and switching back to bf16 captures again;
  * the extra-MSA stack (tied-query ingoing attention) under shard_alphafold2 with its own graph;
  * shard_alphafold2 end to end (default and pair_rows) and recycle() with templates, an extra MSA, the angle heads and the
    structure module: every returned tensor bitwise the use_graph=False model's; launches_per_replay is the library launch
    count of one eager trunk forward;
  * the private workspace: eager ops that grow the shared workspace and release_workspace() between replays;
  * memory: the bytes a live trunk graph holds, and that release_all_graphs() returns them."""
import gc
import os
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------------------
# child-process harness: one-rank NCCL group over a FileStore, graphs released before the group is destroyed
# ------------------------------------------------------------------------------------------------------------
def _worker(case, arg, store_path, q):
    import traceback
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    res = {}
    try:
        import torch.distributed as dist
        from alphafold2_b200 import parallel
        torch.cuda.set_device(0)
        dist.init_process_group("nccl", store=dist.FileStore(store_path, 1), rank=0, world_size=1, device_id=DEV)
        try:
            with torch.no_grad():
                res = globals()[case](arg) or {}
        finally:
            parallel.release_all_graphs()
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res = {"error": traceback.format_exc()}
    q.put(res)


def _spawn(case, arg, tmp_path, timeout=600):
    import queue
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_worker, args=(case, arg, str(tmp_path / "store"), q))
    p.start()
    res, waited = None, 0
    try:
        while res is None:
            try:
                res = q.get(timeout=5)
            except queue.Empty:
                waited += 5
                if not p.is_alive():                       # died without a result (a crash in NCCL init, say): fail now
                    try:
                        res = q.get(timeout=5)
                    except queue.Empty:
                        res = {"error": f"the child process exited with code {p.exitcode} without a result"}
                elif waited >= timeout:
                    res = {"error": f"no result within {timeout} s"}
    finally:
        p.join(timeout=60)
        if p.is_alive():
            p.terminate()
            p.join()
    assert "error" not in res, res["error"]
    return res


# ------------------------------------------------------------------------------------------------------------
# helpers (run in the child)
# ------------------------------------------------------------------------------------------------------------
def _same(a, b):
    if a is None or b is None:
        return a is b
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


class _Captures:
    """Counts the captures of a _GraphedTrunk."""

    def __init__(self, g):
        self.g, self.n = g, 0
        orig = g._capture

        def capture(*a, **k):
            self.n += 1
            return orig(*a, **k)
        g._capture = capture


def _trunk(d, H, dh, N, seed=0, depth=2):
    import alphafold2_b200 as A
    from oracle import evoformer_oracle as O
    torch.manual_seed(seed)
    evo = A.Evoformer(depth=depth, dim=d, seq_len=N, heads=H, dim_head=dh, attn_dropout=0., ff_dropout=0.)
    st = O.randomize_zero_init_({k: v.clone() for k, v in evo.state_dict().items()}, std=0.05)
    evo.load_state_dict(st)
    return evo.to(DEV).eval(), st


def _trunk_inputs(d, N, S, masked, seed):
    g = torch.Generator().manual_seed(seed)
    x, m = torch.randn(1, N, N, d, generator=g), torch.randn(1, S, N, d, generator=g)
    mask = msa_mask = None
    if masked:
        m1 = torch.rand(1, N, generator=g) > 0.15
        m1[:, 0] = True
        mask = m1[:, :, None] & m1[:, None, :]
        msa_mask = torch.rand(1, S, N, generator=g) > 0.1
        msa_mask[:, 0] = True
    return [None if t is None else t.to(DEV) for t in (x, m, mask, msa_mask)]


def _eager(evo, x, m, mask, msa_mask, rows_in=False):
    from alphafold2_b200 import parallel
    return parallel.sharded_evoformer_forward(evo, x, m, mask, msa_mask, None, rows_in=rows_in)


def _replayed(g, cap, captures):
    assert g.failed is None, g.failed
    assert g.graph is not None and cap.n == captures, (g.graph, cap.n, captures)


def _graphed_trunk(d, H, dh, N, seed=0):
    from alphafold2_b200 import parallel
    evo, st = _trunk(d, H, dh, N, seed)
    parallel.shard_evoformer(evo, use_graph=True)
    g = evo._af2_graph
    return evo, st, g, _Captures(g)


def _check_replay(evo, g, cap, captures, inputs, what):
    got = evo(*inputs[:2], mask=inputs[2], msa_mask=inputs[3])
    _replayed(g, cap, captures)
    want = _eager(evo, *inputs)
    assert _same(got[0], want[0]) and _same(got[1], want[1]), f"{what}: the replay is not bitwise the eager schedule"
    return got


# ------------------------------------------------------------------------------------------------------------
# cases (run in the child)
# ------------------------------------------------------------------------------------------------------------
def case_trunk(arg):
    from gpu_util import check, to64
    from oracle import evoformer_oracle as O
    d, H, dh, N, S, masked = arg
    evo, st, g, cap = _graphed_trunk(d, H, dh, N)
    inputs = _trunk_inputs(d, N, S, masked, seed=1)
    first = _check_replay(evo, g, cap, 1, inputs, "capturing call")
    second = _check_replay(evo, g, cap, 1, inputs, "replay")
    assert _same(first[0], second[0]) and _same(first[1], second[1])
    cpu = [None if t is None else t.cpu() for t in inputs]
    rx, rm = O.evoformer(to64(st), "", cpu[0].double(), cpu[1].double(), H, 2, cpu[2], cpu[3])
    check(f"graph_replay/d{d}N{N}S{S}/x", second[0], rx)
    check(f"graph_replay/d{d}N{N}S{S}/m", second[1], rm)


def case_new_inputs(arg):
    d, H, dh, N, S = arg
    evo, _, g, cap = _graphed_trunk(d, H, dh, N)
    a = _trunk_inputs(d, N, S, True, seed=1)
    _check_replay(evo, g, cap, 1, a, "capture")
    b = _trunk_inputs(d, N, S, True, seed=2)                         # new tensors, new values, new masks
    assert not _same(b[2], a[2]) and not _same(b[3], a[3])
    _check_replay(evo, g, cap, 1, b, "new tensors")
    for k, t in enumerate(_trunk_inputs(d, N, S, True, seed=3)):     # the held tensors (a) changed in place
        a[k].copy_(t)
    _check_replay(evo, g, cap, 1, a, "held tensors changed in place")
    for k, t in enumerate(_trunk_inputs(d, N, S, True, seed=4)):     # other tensors (b) changed in place
        b[k].copy_(t)
    _check_replay(evo, g, cap, 1, b, "other tensors changed in place")
    c = _trunk_inputs(d, N, S, False, seed=5)                        # masks None: another signature
    _check_replay(evo, g, cap, 2, c, "no masks")
    _check_replay(evo, g, cap, 3, b, "masks again")


def case_weights(arg):
    import alphafold2_b200 as A
    d, H, dh, N, S = arg
    evo, st, g, cap = _graphed_trunk(d, H, dh, N)
    inputs = _trunk_inputs(d, N, S, True, seed=1)
    base = _check_replay(evo, g, cap, 1, inputs, "capture")
    evo.load_state_dict({k: v * 0.9 + 0.01 if torch.is_floating_point(v) else v for k, v in st.items()})
    out = _check_replay(evo, g, cap, 2, inputs, "load_state_dict")
    assert not _same(out[0], base[0])
    params = [p for p in evo.parameters() if p.dim() == 2]
    p = params[len(params) // 2]
    p.copy_(p * 1.5)                                                 # bumps p._version
    out2 = _check_replay(evo, g, cap, 3, inputs, "p.copy_")
    assert not _same(out2[0], out[0])
    version = p._version
    p.data.add_(0.25)
    assert p._version == version                                     # only invalidate_packed tells the trunk
    A.invalidate_packed(evo)
    out3 = _check_replay(evo, g, cap, 4, inputs, "p.data.add_ + invalidate_packed")
    assert not _same(out3[0], out2[0])
    A.set_precision(evo, "strict")
    with pytest.raises(NotImplementedError):
        evo(*inputs[:2], mask=inputs[2], msa_mask=inputs[3])
    assert g.failed is None, g.failed
    A.set_precision(evo, "bf16")
    out4 = _check_replay(evo, g, cap, 4, inputs, "back to bf16")      # the bf16 signature of before: its graph
    assert _same(out4[0], out3[0]) and _same(out4[1], out3[1])


def _model(n, **kw):
    import test_gpu_recycle_loop as RL
    return RL._model(d=128, depth=2, sdepth=2, n=n, predict_angles=True, **kw)


def case_extra_msa(arg):
    from alphafold2_b200 import parallel
    import test_gpu_sharded_model_ranks as H
    n, S = arg
    model = _model(n)
    parallel.shard_alphafold2(model, use_graph=True)
    stack = model.extra_msa_evoformer
    assert any(b.layer[0].triangle_attention_ingoing.global_query_attn for b in stack.layers)
    g, cap = stack._af2_graph, _Captures(stack._af2_graph)
    seq, mask, kw = H._model_inputs(128, n, S, 1)
    extra_m, em = model.extra_msa_inputs(kw["msa"], kw["extra_msa_mask"])
    x_mask = mask[:, :, None] & mask[:, None, :]
    for seed in (1, 2):
        x = torch.randn(1, n, n, 128, device=DEV, generator=torch.Generator(DEV).manual_seed(seed))
        got = stack(x, extra_m, mask=x_mask, msa_mask=em)
        _replayed(g, cap, 1)
        want = _eager(stack, x, extra_m, x_mask, em)
        assert _same(got[0], want[0]) and _same(got[1], want[1]), seed


def _flat(out):
    import test_gpu_recycle_loop as RL
    return RL._flat(out)


def case_end_to_end(arg):
    from alphafold2_b200 import _lib, parallel
    import alphafold2_b200 as A
    import test_gpu_sharded_model_ranks as H
    n, S, T = arg
    graphed, eager = _model(n), _model(n)
    seq, mask, kw = H._model_inputs(128, n, S, T)
    msa, rec0 = kw.pop("msa"), kw.pop("recyclables")
    kw["mask"] = mask
    flags = dict(return_confidence=True, return_recyclables=True, return_aux_logits=True)
    res = {}
    for pair_rows in (False, True):
        parallel.shard_alphafold2(graphed, use_graph=True, pair_rows=pair_rows)
        parallel.shard_alphafold2(eager, use_graph=False, pair_rows=pair_rows)
        trunks = [(graphed.net._af2_graph, "trunk"), (graphed.extra_msa_evoformer._af2_graph, "extra-MSA stack")]
        for name, run in (("forward", lambda m: m(seq, msa, recyclables=rec0, **kw, **flags)),
                          ("recycle", lambda m: A.recycle(m, seq, msa, num_recycles=2, recyclables=rec0, **kw, **flags))):
            got, want = _flat(run(graphed)), _flat(run(eager))
            assert sorted(got) == sorted(want), (name, sorted(got), sorted(want))
            bad = [k for k in want if not _same(got[k], want[k])]
            assert not bad, f"pair_rows={pair_rows} {name}: not bitwise the eager schedule: {bad}"
            for g, what in trunks:
                assert g.failed is None and g.graph is not None, (what, g.failed)
                assert g.key[-1] is pair_rows, (what, g.key[-1])            # rows_in: the rows trunk's own signature
        for g, what in trunks:
            lib = _lib.load()
            n0 = lib.af2_launch_count()
            g._eager(*g.inputs, rows_in=g.key[-1])
            torch.cuda.synchronize()
            assert g.launches_per_replay == lib.af2_launch_count() - n0, (what, pair_rows, g.launches_per_replay)
            res[(pair_rows, what)] = g.launches_per_replay
    return res


def case_private_workspace(arg):
    from alphafold2_b200 import ops
    d, H, dh, N, S = arg
    evo, _, g, cap = _graphed_trunk(d, H, dh, N)
    inputs = _trunk_inputs(d, N, S, True, seed=1)
    _check_replay(evo, g, cap, 1, inputs, "capture")
    big, _ = _trunk(d, H, dh, 2 * N, seed=3, depth=1)                 # an unsharded trunk at twice N: a larger workspace
    bx = _trunk_inputs(d, 2 * N, S, True, seed=2)
    for round_ in range(2):
        big(*bx[:2], mask=bx[2], msa_mask=bx[3])
        ops.release_workspace(DEV)
        junk = torch.full((1 << 28,), float("nan"), device=DEV)      # 1 GiB of NaN over what was freed
        del junk
        new = _trunk_inputs(d, N, S, True, seed=10 + round_)
        _check_replay(evo, g, cap, 1, new, f"replay {round_} after the shared workspace grew and was released")


def case_memory(arg):
    from alphafold2_b200 import ops, parallel
    d, H, dh, N, S = arg
    evo, _, g, cap = _graphed_trunk(d, H, dh, N)
    inputs = _trunk_inputs(d, N, S, True, seed=1)
    _eager(evo, *inputs)                                              # packs the weights
    ops.release_workspace(DEV)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    alloc0, reserved0 = torch.cuda.memory_allocated(DEV), torch.cuda.memory_reserved(DEV)
    out = _check_replay(evo, g, cap, 1, inputs, "capture")
    del out
    ops.release_workspace(DEV)                                        # the shared one of the eager comparison run
    gc.collect()
    torch.cuda.synchronize()
    alloc1, reserved1 = torch.cuda.memory_allocated(DEV), torch.cuda.memory_reserved(DEV)
    nb = lambda ts: sum(t.numel() * t.element_size() for t in ts if t is not None)  # noqa: E731
    held = dict(inputs=nb(g.inputs), outputs=nb(g.outputs), workspace=nb(g.ws.values()), allocated=alloc1 - alloc0,
                reserved=reserved1 - reserved0, pair_rows_bytes=parallel.pair_rows_bytes(N, S, d, H, dh, 1))
    del inputs
    parallel.release_all_graphs()
    ops.release_workspace(DEV)
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    alloc2, reserved2 = torch.cuda.memory_allocated(DEV), torch.cuda.memory_reserved(DEV)
    assert g.graph is None
    assert alloc2 - alloc0 <= 64 << 10, (alloc0, alloc2)
    held.update(after_release_allocated=alloc2 - alloc0, after_release_reserved=reserved2 - reserved0)
    return held


TRUNK_CASES = [(64, 2, 32, 48, 8, True), (128, 4, 32, 64, 4, False), (256, 8, 64, 136, 40, True), (64, 2, 32, 24, 40, True)]


@pytest.mark.parametrize("d,H,dh,N,S,masked", TRUNK_CASES)
def test_trunk_replay_is_eager_bitwise(tmp_path, d, H, dh, N, S, masked):
    _spawn("case_trunk", (d, H, dh, N, S, masked), tmp_path)


def test_replay_reads_new_inputs(tmp_path):
    _spawn("case_new_inputs", (64, 2, 32, 48, 8), tmp_path)


def test_weight_changes_recapture(tmp_path):
    _spawn("case_weights", (64, 2, 32, 48, 8), tmp_path)


def test_extra_msa_stack_replay(tmp_path):
    _spawn("case_extra_msa", (40, 4), tmp_path)


def test_shard_alphafold2_end_to_end_replay(tmp_path):
    res = _spawn("case_end_to_end", (40, 4, 2), tmp_path, timeout=900)
    print("launches per replay:", res)


def test_private_workspace_survives_shared_growth(tmp_path):
    _spawn("case_private_workspace", (64, 2, 32, 48, 8), tmp_path)


@pytest.mark.parametrize("d,H,dh,N,S", [(128, 4, 32, 128, 16), (256, 8, 32, 256, 32)])
def test_graph_memory_is_returned(tmp_path, d, H, dh, N, S):
    res = _spawn("case_memory", (d, H, dh, N, S), tmp_path)
    mib = {k: round(v / 2**20, 3) for k, v in res.items()}
    print(f"live trunk graph, d {d} N_res {N} S {S}, depth 2, one rank (MiB): {mib}")
