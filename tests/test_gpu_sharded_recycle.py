"""-m gpu: alphafold2_b200.recycle on sharded models against the caller's own recycling loop, with P ranks on ONE GPU (the
harness of tests/test_gpu_sharded_structure_rows.py: P processes on cuda:0 in a gloo group, collectives staged through host
memory), at P = 2 (N_res 40) and P = 3 (N_res 43, pair shards 15 / 14 / 14), with two templates, template angles, an extra
MSA, masks, the angle heads with a symmetrised omega and the structure module, for three modes: shard_evoformer(model)
(the template branch whole on every rank), shard_alphafold2(model) and shard_alphafold2(model, pair_rows=True).  Checks on
every rank:
  * every returned tensor (coordinates, confidence, the distogram and angle logits, rows or whole, every field of
    ret.recyclables) and ret.pair_rows bitwise the loop's, at num_recycles 3 with an initial recyclables, and at num_recycles 1
    under every return flag combination;
  * that the template pair stack runs once per template and prediction when model.last_template_reuse is True, and once per
    template and iteration when it is False (a counter around parallel.sharded_template_pair_stack, or around
    model.template_pair_stack where the branch runs whole);
  * that the reuse rule is collective in the sharded modes: with one rank's rule refusing, every rank takes the path without
    reuse, with the same bits (under shard_evoformer the branch has no collective and each rank decides for itself);
  * peak allocated memory per process: with the rule refusing, recycle peaks no higher than the loop (it only frees the
    previous iteration's outputs earlier); with reuse, no higher than the loop plus the kept template rows.
Not covered here: the peer-store exchange, NCCL and graph replay (they need one GPU per rank)."""
import gc
import os

import pytest
import torch

import test_gpu_sharded_structure_rows as SR

pytestmark = pytest.mark.gpu

D, S, T = 128, 4, 2
MODES = ("evoformer", "default", "rows")


class _Count:
    def __init__(self, fn):
        self.fn, self.calls = fn, 0

    def __call__(self, *a, **k):
        self.calls += 1
        return self.fn(*a, **k)


def _flat(out):
    import test_gpu_recycle_loop as RL
    res = RL._flat(out)
    if not torch.is_tensor(out) and not torch.is_tensor(out[1]) and getattr(out[1], "pair_rows", None) is not None:
        res["pair_rows"] = torch.tensor(out[1].pair_rows)
    return res


def _bad(got, want):
    from test_gpu_recycle_loop import _bits
    return sorted(set(got) ^ set(want)) + sorted(k for k in set(got) & set(want) if got[k].shape != want[k].shape or
                                                 got[k].dtype != want[k].dtype or not torch.equal(_bits(got[k]), _bits(want[k])))


def _run(rank, P, case):
    import itertools
    import alphafold2_b200 as A
    from alphafold2_b200 import ops, parallel
    import test_gpu_recycle_loop as RL
    import test_gpu_sharded_model_ranks as H
    n = case
    model = RL._model(d=D, depth=2, sdepth=2, n=n, predict_angles=True, symmetrize_omega=True)
    seq, mask, kw = H._model_inputs(D, n, S, T)
    msa, rec0 = kw.pop("msa"), kw.pop("recyclables")
    kw["mask"] = mask
    dev = torch.device("cuda", 0)
    on = parallel.shard_offsets(n, P)
    rows = on[rank + 1] - on[rank]
    out = {}

    def compare(R, **extra):
        want = _flat(RL.manual_loop(model, seq, msa, R, **kw, **extra))
        cnt.calls = 0
        got = _flat(A.recycle(model, seq, msa, num_recycles=R, **kw, **extra))
        return _bad(got, want), cnt.calls, model.last_template_reuse

    def refuse_on(r_refuse):
        """Make the mode's reuse rule refuse on rank r_refuse (every rank when None); returns the undo."""
        mod, name = (ops, "template_reuse_fits") if mode == "evoformer" else (parallel, "template_reuse_rows_fits")
        orig = getattr(mod, name)
        setattr(mod, name, lambda *a, **k: False if r_refuse in (None, rank) else orig(*a, **k))
        return lambda: setattr(mod, name, orig)

    def peak(fn):
        gc.collect()
        ops.release_workspace(dev)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        res = fn()
        torch.cuda.synchronize()
        del res
        return torch.cuda.max_memory_allocated()

    for mode in MODES:
        if mode == "evoformer":
            parallel.shard_evoformer(model, use_graph=False)
            cnt = _Count(model.template_pair_stack)
            model.template_pair_stack = cnt
            per_iter, kept = 1, T * n * n * (4 * D + 1)             # the branch runs whole: one stack call for G = T templates
        else:
            parallel.shard_alphafold2(model, use_graph=False, pair_rows=mode == "rows")
            cnt = _Count(parallel.sharded_template_pair_stack)
            parallel.sharded_template_pair_stack = cnt
            per_iter, kept = T, T * rows * n * (4 * D + 1)
        res = out[mode] = {}
        try:
            all_flags = dict(return_confidence=True, return_recyclables=True, return_aux_logits=True)
            res["r3"] = compare(3, recyclables=rec0, **all_flags) + (per_iter,)
            res["flags"] = {f: compare(1, **dict(zip(RL.FLAGS, f))) for f in itertools.product((False, True), repeat=3)}
            undo = refuse_on(1)
            try:
                res["refused_on_1"] = compare(1, **all_flags) + (2 * per_iter if mode != "evoformer" or rank == 1 else per_iter,)
            finally:
                undo()
            peaks = {}
            for reuse in (False, True):
                undo = (lambda: None) if reuse else refuse_on(None)
                try:
                    runs = {"manual": lambda: RL.manual_loop(model, seq, msa, 1, return_confidence=True, **kw),
                            "recycle": lambda: A.recycle(model, seq, msa, num_recycles=1, return_confidence=True, **kw)}
                    for name in ("manual", "recycle") * 2:
                        peaks[(reuse, name)] = peak(runs[name])
                    peaks[(reuse, "reuse")] = model.last_template_reuse
                finally:
                    undo()
            res["peaks"] = peaks
            res["kept"] = kept
        finally:
            if mode == "evoformer":
                del model.template_pair_stack
            else:
                parallel.sharded_template_pair_stack = cnt.fn
    return out


def _worker(rank, P, port, case, q):
    import datetime
    import sys
    import traceback
    import torch.distributed as dist
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [root, os.path.join(root, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        from test_gpu_sharded_ranks_uneven import _stage_collectives_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            SR._stage_broadcast_through_host()
            with torch.no_grad():
                res.update(_run(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


@pytest.mark.parametrize("P,n", [(2, 40), (3, 43)])
def test_sharded_recycle_is_the_manual_loop_one_gpu(monkeypatch, P, n):
    monkeypatch.setattr(SR, "_worker", _worker)
    for r in SR._spawn(P, n):
        for mode in MODES:
            res = r[mode]
            bad, calls, reuse, per_iter = res["r3"]
            assert bad == [] and reuse is True, (r["rank"], mode, bad, reuse)
            assert calls == per_iter, (r["rank"], mode, calls)
            for f, (bad, calls, reuse) in res["flags"].items():
                assert bad == [] and reuse is True and calls == per_iter, (r["rank"], mode, f, bad, calls, reuse)
            bad, calls, reuse, want_calls = res["refused_on_1"]
            collective = mode != "evoformer"
            assert bad == [], (r["rank"], mode, bad)
            assert reuse is (False if collective or r["rank"] == 1 else True), (r["rank"], mode, reuse)
            assert calls == want_calls, (r["rank"], mode, calls, want_calls)
            pk = res["peaks"]
            print(f"  P={P} N_res={n} rank {r['rank']} {mode}: peak allocated without reuse: loop {pk[(False, 'manual')] / 2**20:.2f} "
                  f"MiB, recycle {pk[(False, 'recycle')] / 2**20:.2f} MiB; with reuse: loop {pk[(True, 'manual')] / 2**20:.2f} MiB, "
                  f"recycle {pk[(True, 'recycle')] / 2**20:.2f} MiB (kept template rows {res['kept'] / 2**20:.2f} MiB)")
            assert pk[(False, "reuse")] is False and pk[(True, "reuse")] is True
            assert pk[(False, "recycle")] <= pk[(False, "manual")], (r["rank"], mode, pk)
            assert pk[(True, "recycle")] <= pk[(True, "manual")] + res["kept"], (r["rank"], mode, pk, res["kept"])
