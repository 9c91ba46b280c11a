"""-m gpu: alphafold2_b200.recycle against the caller's own recycling loop

    coords, ret = model(seq, msa, **kw, return_aux_logits=True, return_recyclables=True)
    for _ in range(num_recycles):
        coords, ret = model(seq, msa, **kw, recyclables=ret.recyclables, return_aux_logits=True, return_recyclables=True)

with the caller's return flags on the last call.  Every returned tensor (coordinates, confidence, distogram, angle logits, every
field of ret.recyclables) must be bitwise the loop's, never a tolerance: recycle runs the same kernels on the same inputs and
only keeps the template pair stack's output or frees tensors earlier.  Covered: batch 2 with padded masks, num_recycles 0, 1
and 3, templates with template angles (the stack kept, refused by the reuse rule, and run in groups under a small budget), an
extra MSA beside templates, the angle heads with a symmetrised omega, strict mode, an initial recyclables and every return
flag combination; the refusals; the peak memory against the loop; P = 2 ranks of shard_alphafold2 on one GPU."""
import itertools
import math
import os

import pytest
import torch

import alphafold2_b200 as A
from alphafold2_b200 import ops
from oracle import evoformer_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
FLAGS = ("return_confidence", "return_recyclables", "return_aux_logits")


def _model(d=128, depth=2, sdepth=2, n=24, precision="bf16", predict_coords=True, attach=True, **kw):
    torch.manual_seed(0)
    model = A.Alphafold2(dim=d, depth=depth, heads=2, dim_head=32, max_seq_len=n, extra_msa_evoformer_layers=1,
                         templates_embed_layers=2, predict_coords=predict_coords, structure_module_depth=sdepth,
                         structure_module_heads=2, **kw)
    if attach:
        A.attach_structure_module(model)
    model.load_state_dict(O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    return A.set_precision(model.to(DEV).eval(), precision)


def _inputs(d, b=2, n=24, S=3, T=2, extra=False, angles=True, recyclables=False):
    g = torch.Generator().manual_seed(7)
    seq = torch.randint(0, 21, (b, n), generator=g)
    msa = torch.randint(0, 21, (b, S, n), generator=g)
    mask = torch.ones(b, n, dtype=torch.bool)
    mask[0, -n // 4:] = False                                             # padding
    msa_mask = torch.rand(b, S, n, generator=g) > 0.1
    msa_mask[:, 0] = mask
    kw = dict(mask=mask, msa_mask=msa_mask)
    if T:
        tm = torch.rand(b, T, n, generator=g) > 0.1
        if T > 1:
            tm[1, -1] = False                                             # a template with no valid residue
        kw.update(templates_feats=torch.randn(b, T, n, n, 32, generator=g), templates_mask=tm)
        if angles:
            kw["templates_angles"] = torch.randn(b, T, n, 55, generator=g)
    if extra:
        kw.update(extra_msa=torch.randint(0, 21, (b, S, n), generator=g), extra_msa_mask=torch.rand(b, S, n, generator=g) > 0.1)
    kw = {k: v.to(DEV) for k, v in kw.items()}
    if recyclables:
        kw["recyclables"] = A.Recyclables(torch.randn(b, n, 3, generator=g).to(DEV) * 8, torch.randn(b, n, d, generator=g).to(DEV),
                                          torch.randn(b, n, n, d, generator=g).to(DEV))
    return seq.to(DEV), msa.to(DEV), kw


def manual_loop(model, seq, msa, num_recycles, **kw):
    flags = {k: kw.pop(k) for k in FLAGS if k in kw}
    if num_recycles == 0:
        return model(seq, msa, **kw, **flags)
    coords, ret = model(seq, msa, **kw, return_aux_logits=True, return_recyclables=True)
    kw.pop("recyclables", None)
    for _ in range(num_recycles - 1):
        coords, ret = model(seq, msa, **kw, recyclables=ret.recyclables, return_aux_logits=True, return_recyclables=True)
    return model(seq, msa, **kw, recyclables=ret.recyclables, **flags)


def _flat(out):
    """A forward's return value as {name: cpu tensor}, in the form Alphafold2.forward gives it."""
    if torch.is_tensor(out):
        res = {"coords": out}
    elif torch.is_tensor(out[1]):
        res = {"coords": out[0], "confidence": out[1]}
    else:
        ret = out[1]
        res = {"coords": out[0], "distance": ret.distance}
        for k in ("theta_logits", "phi_logits", "omega_logits"):
            if getattr(ret, k, None) is not None:
                res[k] = getattr(ret, k)
        if ret.recyclables is not None:
            r = ret.recyclables
            res.update(rec_coords=r.coords, rec_single=r.single_msa_repr_row, rec_pair=r.pairwise_repr)
    return {k: v.detach().cpu() for k, v in res.items()}


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _assert_same(got, want):
    assert sorted(got) == sorted(want)
    bad = [k for k in want if got[k].shape != want[k].shape or got[k].dtype != want[k].dtype or
           not torch.equal(_bits(got[k]), _bits(want[k]))]
    assert not bad, f"not bitwise the manual loop: {bad}"


class _Spy:
    """Counts model.template_pair_stack calls and keeps the first one's t with a copy of it."""

    def __init__(self, model):
        self.fn, self.calls, self.first = model.template_pair_stack, 0, None
        model.template_pair_stack = self

    def __call__(self, *a, **k):
        out = self.fn(*a, **k)
        self.calls += 1
        if self.first is None:
            self.first = (out[0], out[0].clone())
        return out


def _compare(model, seq, msa, num_recycles, **kw):
    with torch.no_grad():
        want = _flat(manual_loop(model, seq, msa, num_recycles, **kw))
        spy = _Spy(model)
        try:
            got = _flat(A.recycle(model, seq, msa, num_recycles=num_recycles, **kw))
        finally:
            del model.template_pair_stack
    _assert_same(got, want)
    return spy


CASES = {
    "templates": dict(model=dict(), inputs=dict()),
    "no_templates_d64": dict(model=dict(d=64, depth=1, sdepth=1), inputs=dict(T=0)),
    "extra_msa_templates": dict(model=dict(), inputs=dict(extra=True)),
    "angles_symmetrized": dict(model=dict(predict_angles=True, symmetrize_omega=True), inputs=dict(T=1)),
    "initial_recyclables": dict(model=dict(d=64, depth=1, sdepth=1), inputs=dict(recyclables=True)),
    "strict": dict(model=dict(d=64, depth=1, sdepth=1, precision="strict"), inputs=dict(T=2)),
}


@pytest.mark.parametrize("case,num_recycles", [(c, r) for c in CASES for r in (0, 1, 3) if not (c == "strict" and r == 3)])
def test_recycle_is_the_manual_loop(case, num_recycles):
    c = CASES[case]
    model = _model(**c["model"])
    seq, msa, kw = _inputs(model.dim, **c["inputs"])
    spy = _compare(model, seq, msa, num_recycles, return_aux_logits=True, return_recyclables=True, **kw)
    if "templates_feats" in kw:
        if num_recycles:
            assert model.last_template_reuse is True
            assert spy.calls == 1
            t, t0 = spy.first
            assert torch.equal(_bits(t), _bits(t0)), "the kept t changed"
        else:
            assert spy.calls == 1


@pytest.mark.parametrize("flags", list(itertools.product((False, True), repeat=3)))
def test_every_return_flag_combination(flags):
    model = _model(d=64, depth=1, sdepth=1)
    seq, msa, kw = _inputs(model.dim, T=1)
    _compare(model, seq, msa, 1, **dict(zip(FLAGS, flags)), **kw)


def test_no_reuse_when_the_rule_refuses(monkeypatch):
    """ops.template_reuse_fits given no budget refuses: every iteration runs the pair stack, with the same bits."""
    fits = ops.template_reuse_fits
    seen = []

    def refuse(*a):
        seen.append(a[-1])
        return fits(*a[:-1], 0)

    monkeypatch.setattr(ops, "template_reuse_fits", refuse)
    model = _model()
    seq, msa, kw = _inputs(model.dim, extra=True)
    spy = _compare(model, seq, msa, 3, return_aux_logits=True, return_recyclables=True, **kw)
    assert len(seen) == 1 and seen[0] > 0
    assert model.last_template_reuse is False
    assert spy.calls == 4


def test_no_reuse_when_the_templates_run_in_groups(monkeypatch):
    """A budget under which the template branch runs in groups (G < T) but the trunk still runs whole: no reuse, same bits."""
    b, T, n, S = 2, 3, 24, 3
    model = _model(n=n)
    seq, msa, kw = _inputs(model.dim, b=b, n=n, S=S, T=T)
    d, H, DH = model.dim, 2, 32
    lo = max(ops.pair_block_bytes(b, n, S + T, d, H, DH, n), ops.template_branch_bytes(b, T, 1, n, d, H, DH, "bf16"))
    hi = ops.template_branch_bytes(b, T, T, n, d, H, DH, "bf16")
    assert lo < hi
    budget = int(((lo + hi) // 2) / 0.85) + 1
    monkeypatch.setattr(ops, "device_budget", lambda device: budget)
    spy = _compare(model, seq, msa, 2, return_aux_logits=True, return_recyclables=True, **kw)
    G = model.last_template_group
    assert G < T and model.last_template_reuse is False
    assert spy.calls == 3 * math.ceil(T / G)


def _snapshot(seq, msa, kw):
    out = [seq.clone(), msa.clone()]
    for v in kw.values():
        out += [t.clone() for t in ((v.coords, v.single_msa_repr_row, v.pairwise_repr) if isinstance(v, A.Recyclables) else (v,))]
    return out


@pytest.mark.parametrize("what", ["negative", "no_coords", "return_trunk", "unattached"])
def test_refusals_before_any_launch(what):
    lib = ops._lib.load()
    model = _model(d=64, depth=1, sdepth=1, predict_coords=what != "no_coords", attach=what != "unattached")
    seq, msa, kw = _inputs(model.dim, T=1, recyclables=True)
    before = _snapshot(seq, msa, kw)
    torch.cuda.synchronize()
    n0 = lib.af2_launch_count()
    err, match = (NotImplementedError, "attach_structure_module") if what == "unattached" else (ValueError, None)
    with pytest.raises(err, match=match), torch.no_grad():
        A.recycle(model, seq, msa, num_recycles=-1 if what == "negative" else 2, return_trunk=what == "return_trunk", **kw)
    torch.cuda.synchronize()
    assert lib.af2_launch_count() == n0
    assert all(torch.equal(a, b) for a, b in zip(before, _snapshot(seq, msa, kw)))


def test_peak_memory_below_the_manual_loop(monkeypatch):
    """N_res 768, d 128, one MSA row, with the device budget set so that the pair track runs in bands of 256 rows: the pair
    tensor (288 MiB) then outweighs the workspace.  The manual loop holds the previous pair tensor through the whole second
    forward; recycle frees it once read."""
    b, n, d, S = 1, 768, 128, 1
    model = _model(d=d, depth=1, sdepth=1, n=n)
    seq, msa, kw = _inputs(d, b=b, n=n, S=S, T=0)
    banded = ops.pair_block_bytes(b, n, S, d, 2, 32, 256)
    assert ops.pair_block_bytes(b, n, S, d, 2, 32, 512) > banded
    budget = int((banded + (1 << 20)) / 0.85) + 1
    monkeypatch.setattr(ops, "device_budget", lambda device: budget)
    runs = {"manual": lambda: manual_loop(model, seq, msa, 1, return_confidence=True, **kw),
            "recycle": lambda: A.recycle(model, seq, msa, num_recycles=1, return_confidence=True, **kw)}
    peaks = {}
    for name in ("manual", "recycle") * 2:
        # the workspace is keyed by the tensors' device (cuda:0, not "cuda"); one an earlier test left at a whole block's
        # size would make the trunk run whole (_block_bands) whatever the budget
        ops.release_workspace(seq.device)
        assert not ops.workspace_holds(seq.device, 1)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            out = runs[name]()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated()
        del out
    assert model.net.last_pair_band == 256
    pair = 4 * b * n * n * d
    print(f"recycle memory at N_res {n}, d {d}, one MSA row, pair bands of 256: peak allocated manual loop "
          f"{peaks['manual'] / 2**20:.1f} MiB, recycle {peaks['recycle'] / 2**20:.1f} MiB, saving "
          f"{(peaks['manual'] - peaks['recycle']) / 2**20:.1f} MiB, pair tensor {pair / 2**20:.1f} MiB")
    assert peaks["manual"] - peaks["recycle"] >= 0.9 * pair


# ------------------------------------------------------------------------------------------------------------- sharded
def _run_sharded(rank, P, case):
    import test_gpu_sharded_model_ranks as H
    from alphafold2_b200 import parallel
    n, S, T = case
    model = _model(d=128, depth=2, sdepth=2, n=n)
    seq, mask, kw = H._model_inputs(128, n, S, T)
    flags = dict(return_aux_logits=True, return_recyclables=True)
    res = {}
    for rows in (False, True):
        parallel.shard_alphafold2(model, use_graph=False, pair_rows=rows)
        want = _flat(manual_loop(model, seq, kw["msa"], 2, mask=mask, **{k: v for k, v in kw.items() if k != "msa"}, **flags))
        got = _flat(A.recycle(model, seq, kw["msa"], num_recycles=2, mask=mask, **{k: v for k, v in kw.items() if k != "msa"},
                              **flags))
        res[f"pair_rows={rows}"] = sorted(k for k in want if k not in got or not torch.equal(_bits(got[k]), _bits(want[k])))
    return res


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
        from test_gpu_sharded_structure_rows import _stage_broadcast_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            _stage_broadcast_through_host()
            with torch.no_grad():
                res.update(_run_sharded(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


def test_sharded_recycle_is_the_manual_loop_one_gpu(monkeypatch):
    """P = 2 processes on one GPU (the harness of test_gpu_sharded_structure_rows.py): recycle on a shard_alphafold2 model,
    default and pair_rows, is bitwise the manual loop on every rank."""
    import test_gpu_sharded_structure_rows as SR
    monkeypatch.setattr(SR, "_worker", _worker)
    for r in SR._spawn(2, (40, 4, 1)):
        assert r["pair_rows=False"] == [] and r["pair_rows=True"] == [], r
