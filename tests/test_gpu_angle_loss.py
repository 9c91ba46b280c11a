"""-m gpu: the angle-head labels and loss (utils.get_bucketed_angle_matrices, utils.angle_loss, parallel.angle_loss_rows)
against the fp64 oracle (oracle/angle_loss_oracle.py).

  * labels bitwise the oracle's: random backbones with A 3 and 14, planar residues whose theta and omega are exactly 0 or +pi,
    NaN atoms, [N, A, 3] input, mask None, several bucket counts;
  * each head's loss within the distogram oracle's bound (its CPU controls are in tests/test_oracle_angle_loss.py);
  * the F.cross_entropy quirks: an in-range ignore_index, nothing counted (NaN), mask None;
  * the contract: reproducible bits, two launches and no host synchronisation, 48 bytes per (element, row) above the inputs,
    one head past 2^31 elements, and refusals before any launch;
  * per-row partials of any split of the rows combine bitwise to the whole; and parallel.angle_loss_rows on the rows of a
    shard_alphafold2(pair_rows=True) forward with predict_angles=True at P = 2, 3 and 4 on one GPU returns on every rank
    bitwise utils.angle_loss of the gathered logits."""
import math
import os
import queue

import pytest
import torch

from oracle import angle_loss_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NB = (25, 13, 25)


def _u():
    from alphafold2_b200 import utils
    return utils


def _launches():
    from alphafold2_b200 import _lib
    return _lib.load().af2_launch_count()


def backbone(b, n, g, A=3, scale=6.0):
    """[b, n, A, 3]: CA on a random walk in a box, N and C at bond lengths in random directions, atoms 3.. random"""
    step = torch.randn(b, n, 3, generator=g, dtype=torch.float64)
    ca = (step / step.norm(dim=-1, keepdim=True) * 3.8).cumsum(1) * 0.5 + torch.randn(b, n, 3, generator=g, dtype=torch.float64) * scale
    d = torch.randn(b, n, 2, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    bb = torch.stack([ca + 1.46 * d[:, :, 0], ca, ca + 1.52 * d[:, :, 1]], 2)
    if A > 3:
        bb = torch.cat([bb, ca[:, :, None] + torch.randn(b, n, A - 3, 3, generator=g, dtype=torch.float64) * 2], 2)
    return bb.float()


def planar(n, g):
    """[1, n, 3, 3] residues in the plane z = 2^60: each virtual CB's offset from the plane is below half an ulp of 2^60, so
    every CB lies in the plane too and theta and omega are exactly 0 or +pi (one contact in three is cis or trans)"""
    xy = torch.randn(n, 3, 2, generator=g) * 6
    xy[:, 1] = xy[:, 0] + torch.randn(n, 2, generator=g)
    bb = torch.zeros(1, n, 3, 3)
    bb[0, :, :, :2] = xy
    bb[..., 2] = 2.0 ** 60
    return bb


def _labels_equal(bb, mask, nb=NB, ii=-100):
    U = _u()
    got = U.get_bucketed_angle_matrices(bb.cuda(), None if mask is None else mask.cuda(), nb, ii)
    want = O.labels(bb, mask, nb, ii)
    for h, (x, y) in enumerate(zip(got, want)):
        assert x.dtype == torch.int64 and x.shape == y.shape
        assert torch.equal(x.cpu(), y), f"head {h}: {(x.cpu() != y).sum().item()} labels differ"
    return want


@pytest.mark.parametrize("b,n,A,nb", [(2, 150, 3, NB), (1, 257, 14, NB), (3, 64, 3, (2, 2, 2)), (2, 90, 4, (37, 7, 64)),
                                      (1, 200, 14, (101, 13, 9))])
def test_labels_vs_oracle(b, n, A, nb):
    g = torch.Generator().manual_seed(n + A)
    bb = backbone(b, n, g, A, scale=4.0)
    bb[-1, n // 3, 1, 0] = float("nan")                         # a missing CA: no contact with anything
    mask = torch.rand(b, n, generator=g) > 0.2
    mask[-1, n // 3] = True
    want = _labels_equal(bb, mask, nb, -7)
    for t, k in zip(want, nb):
        assert (t == k - 1).any() and (t == 0).any()
        assert bool((t[-1, n // 3][mask[-1]] == k - 1).all())
    U = _u()
    flat = U.get_bucketed_angle_matrices(bb[0].cuda(), mask[0].cuda(), nb, -7)
    assert all(f.shape == (n, n) and torch.equal(f.cpu(), w[0]) for f, w in zip(flat, want))
    _labels_equal(bb, None, nb)


def test_planar_labels():
    g = torch.Generator().manual_seed(3)
    bb = planar(120, g)
    th, ph, om, c = O.angles(bb)
    assert set(th[c].unique().tolist()) <= {0.0, math.pi} and set(om[c].unique().tolist()) == {0.0, math.pi}
    lab = _labels_equal(bb, None)
    assert set(lab[0][c].unique().tolist()) <= {11, 23} and set(lab[2][c].unique().tolist()) == {11, 23}


def _check_loss(got, logits, lab, ii=-100):
    for h, (x, l, t) in enumerate(zip((got.theta, got.phi, got.omega), logits, lab)):
        assert x.dim() == 0 and x.dtype == torch.float32 and x.is_cuda
        want = O.loss64(l.cpu(), t.cpu(), ii).item()
        bound = O.loss_bound(l.cpu(), t.cpu(), ii)
        assert abs(x.item() - want) <= bound or (math.isnan(want) and math.isnan(x.item())), (h, x.item(), want, bound)


def _logits(b, n, nb, g, scale=3.0):
    return [torch.randn(b, n, n, k, generator=g) * scale for k in nb]


@pytest.mark.parametrize("b,n,A,nb,scale", [(1, 300, 3, NB, 3.0), (2, 129, 14, NB, 30.0), (3, 64, 3, (2, 3, 2), 3.0),
                                            (1, 77, 4, (64, 13, 200), 2.0), (16, 40, 3, NB, 3.0)])
def test_loss_vs_oracle(b, n, A, nb, scale):
    U = _u()
    g = torch.Generator().manual_seed(b * 1000 + n)
    bb = backbone(b, n, g, A, scale=4.0)
    bb[0, 3, 0, 2] = float("nan")
    mask = torch.rand(b, n, generator=g) > 0.15
    lg = _logits(b, n, nb, g, scale)
    loss = U.angle_loss(*(t.cuda() for t in lg), bb.cuda(), mask.cuda())
    _check_loss(loss, lg, O.labels(bb, mask, nb))


def test_quirks():
    U = _u()
    g = torch.Generator().manual_seed(9)
    b, n = 3, 60
    bb, lg = backbone(b, n, g, scale=3.0), _logits(b, n, NB, g)
    mask = torch.ones(b, n, dtype=torch.bool)
    mask[0, :30] = False
    mask[1, 5:] = False
    bc, lc, mc = bb.cuda(), [t.cuda() for t in lg], mask.cuda()
    for ii in (3, 12, 24, 0, -100, 1000):                          # in range: the bucket drops out too (12 is phi's no contact)
        _check_loss(U.angle_loss(*lc, bc, mc, ii), lg, O.labels(bb, mask, NB, ii), ii)
    _check_loss(U.angle_loss(*lc, bc), lg, O.labels(bb, None, NB))  # mask=None
    nan = U.angle_loss(*lc, bc, torch.zeros_like(mc))                # nothing counts: 0 / 0
    assert all(torch.isnan(t) for t in (nan.theta, nan.phi, nan.omega))
    a, c = U.angle_loss(*lc, bc, None), U.angle_loss(*lc, bc, torch.ones_like(mc))
    assert all(torch.equal(x, y) for x, y in ((a.theta, c.theta), (a.phi, c.phi), (a.omega, c.omega)))


def test_contract_bits_launches_memory():
    U = _u()
    g = torch.Generator().manual_seed(4)
    b, n = 2, 1000
    bb = backbone(b, n, g, 14, scale=10.0).cuda()
    lg = [t.cuda() for t in _logits(b, n, NB, g)]
    mask = (torch.rand(b, n, generator=g) > 0.1).cuda()
    U.angle_loss(*lg, bb, mask)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    k0 = _launches()
    first = U.angle_loss(*lg, bb, mask)
    assert _launches() - k0 == 2
    second = U.angle_loss(*lg, bb, mask)
    torch.cuda.synchronize()
    for h in ("theta", "phi", "omega"):
        assert torch.equal(getattr(first, h).view(torch.int32), getattr(second, h).view(torch.int32))
    assert torch.cuda.max_memory_allocated() - base <= 48 * b * n + 4096
    torch.cuda._sleep(200_000_000)                                  # no host synchronisation
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    U.angle_loss(*lg, bb, mask)
    assert not start.query(), "angle_loss waited for the device"
    torch.cuda.synchronize()


def test_past_2_31_elements():
    """theta with 1024 buckets at N 1500 holds 2.3e9 elements; the fp64 oracle runs on the device in row blocks"""
    U = _u()
    n, nb = 1500, (1024, 13, 25)
    assert n * n * nb[0] > 2 ** 31
    g = torch.Generator().manual_seed(1)
    bb = backbone(1, n, g, scale=8.0)
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[0, -7:] = False
    gd = torch.Generator(device="cuda").manual_seed(1)
    lg = [torch.randn(1, n, n, k, device="cuda", generator=gd) for k in nb]
    loss = U.angle_loss(*lg, bb.cuda(), mask.cuda())
    lab = [t.cuda() for t in O.labels(bb, mask, nb)]
    from oracle import distogram_loss_oracle as D
    for h, got in enumerate((loss.theta, loss.phi, loss.omega)):
        want, bound, k = 0.0, 0.0, 0
        for r0 in range(0, n, 100):
            t = D.terms64(lg[h][:, r0:r0 + 100], lab[h][:, r0:r0 + 100], -100)
            want += t.sum().item()
            k += t.numel()
            bound += D.term_bound(lg[h][:, r0:r0 + 100], lab[h][:, r0:r0 + 100], -100).sum().item()
        want /= k
        assert abs(got.item() - want) <= bound / k + 2 ** -23 * abs(want) + 1e-12, (h, got.item(), want)


def test_refusals():
    U = _u()
    x = torch.randn(1, 8, 3, 3, device="cuda")
    th, ph, om = (torch.randn(1, 8, 8, k, device="cuda") for k in NB)
    m = torch.ones(1, 8, dtype=torch.bool, device="cuda")
    L = U.angle_loss
    bad = [
        (lambda: L(th.cpu(), ph, om, x, m), RuntimeError),
        (lambda: L(th, ph, om, x.cpu(), m), RuntimeError),
        (lambda: L(th, ph.clone().requires_grad_(), om, x, m), RuntimeError),
        (lambda: L(th, ph, om, x.clone().requires_grad_(), m), RuntimeError),
        (lambda: L(th, ph, om, x[:, :7], m), ValueError),
        (lambda: L(th, ph, om, x.expand(2, 8, 3, 3), m), ValueError),
        (lambda: L(th, ph, om, x[:, :, :2], m), ValueError),
        (lambda: L(th, ph, om, x[..., :2], m), ValueError),
        (lambda: L(th, ph, om, x, m[:, :7]), ValueError),
        (lambda: L(th, ph[:, :7], om, x, m), ValueError),
        (lambda: L(th, ph, om[:, :, :7], x, m), ValueError),
        (lambda: L(th, ph, om.expand(2, 8, 8, 25), x, m), ValueError),
        (lambda: L(th[0], ph, om, x, m), ValueError),
        (lambda: L(th[..., :1], ph, om, x, m), ValueError),
        (lambda: L(th, ph, torch.randn(1, 8, 8, 4090, device="cuda"), x, m), ValueError),
        (lambda: L(th[:0], ph[:0], om[:0], x[:0], m[:0]), ValueError),
        (lambda: L(th, ph, om, x, m, ignore_index=-100.0), TypeError),
        (lambda: L(th, ph, om, x, m, ignore_index=True), TypeError),
        (lambda: L(th, ph, om, x, m.float()), TypeError),
        (lambda: U.get_bucketed_angle_matrices(x.cpu(), m.cpu()), RuntimeError),
        (lambda: U.get_bucketed_angle_matrices(x, m, (25, 1, 25)), ValueError),
        (lambda: U.get_bucketed_angle_matrices(x, m, (25, 13)), ValueError),
        (lambda: U.get_bucketed_angle_matrices(x, m, NB, 1.5), TypeError),
        (lambda: U.get_bucketed_angle_matrices(x[:, :, :2], m), ValueError),
        (lambda: U.get_bucketed_angle_matrices(x, m[:, :5]), ValueError),
    ]
    torch.cuda.synchronize()
    k0 = _launches()
    for i, (call, exc) in enumerate(bad):
        with pytest.raises(exc):
            call()
        assert _launches() == k0, f"refusal {i} launched a kernel"


@pytest.mark.parametrize("n,splits", [(97, [48, 49]), (97, [1] * 97), (128, [32, 32, 32, 32]), (60, [7, 20, 33])])
def test_row_partials_any_split(n, splits):
    from alphafold2_b200 import ops
    U = _u()
    g = torch.Generator().manual_seed(n)
    b = 2
    bb = backbone(b, n, g, scale=3.0).cuda()
    lg = [t.cuda() for t in _logits(b, n, NB, g)]
    mask = (torch.rand(b, n, generator=g) > 0.2).cuda()
    whole = ops.angle_xent_rows(*lg, bb, mask, -100)
    parts, r0 = [], 0
    for r in splits:
        parts.append(ops.angle_xent_rows(*(t[:, r0:r0 + r].contiguous() for t in lg), bb, mask, -100, row0=r0))
        r0 += r
    joined = torch.cat(parts, 1)
    assert torch.equal(joined, whole)
    fin = ops.angle_xent_finish(joined.contiguous())
    ref = U.angle_loss(*lg, bb, mask)
    assert torch.equal(fin.view(torch.int32), torch.stack([ref.theta, ref.phi, ref.omega]).view(torch.int32))


# ---- sharded: parallel.angle_loss_rows on the ranks of shard_alphafold2(pair_rows=True), P processes on cuda:0 ----
SHARD_CASES = [(2, 40), (3, 43), (4, 48)]


def _run_rows(rank, P, n):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel, utils
    from oracle import evoformer_oracle as E
    from test_gpu_sharded_ranks_uneven import _digest
    torch.manual_seed(0)
    d = 128
    model = A.Alphafold2(dim=d, depth=1, heads=2, dim_head=32, max_seq_len=n, predict_angles=True, symmetrize_omega=True)
    model.load_state_dict(E.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, n)).cuda()
    msa = torch.randint(0, 21, (1, 3, n)).cuda()
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -n // 8:] = False
    mask = mask.cuda()
    bb = backbone(1, n, torch.Generator().manual_seed(n), 14, scale=3.0).cuda()
    parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)
    with torch.no_grad():
        ret = model(seq, msa, mask=mask)
    heads = (ret.theta_logits, ret.phi_logits, ret.omega_logits)
    rows = parallel.angle_loss_rows(*heads, bb, mask)
    rows_nomask = parallel.angle_loss_rows(*heads, bb, None, ignore_index=5)
    whole = [parallel.gather_pair_rows(t) for t in heads]
    ref = utils.angle_loss(*whole, bb, mask)
    ref_nomask = utils.angle_loss(*whole, bb, None, ignore_index=5)
    flat = lambda r: torch.stack([r.theta, r.phi, r.omega])  # noqa: E731
    return {"digest": _digest(flat(rows).cpu(), flat(rows_nomask).cpu()),
            "equal": torch.equal(flat(rows).view(torch.int32), flat(ref).view(torch.int32))
            and torch.equal(flat(rows_nomask).view(torch.int32), flat(ref_nomask).view(torch.int32)),
            "loss": flat(rows).tolist()}


def _worker(rank, P, port, n, q):
    import datetime
    import sys
    import traceback
    import torch.distributed as dist
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        from test_gpu_sharded_ranks_uneven import _stage_collectives_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            res.update(_run_rows(rank, P, n))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


@pytest.mark.parametrize("P,n", SHARD_CASES)
def test_angle_loss_rows_sharded_one_gpu(P, n):
    import torch.multiprocessing as mp
    from test_gpu_sharded_ranks_uneven import _free_port
    if torch.cuda.is_initialized():
        import gc
        from alphafold2_b200 import ops
        gc.collect()
        ops.release_workspace(torch.device("cuda", 0))
        torch.cuda.empty_cache()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, P, port, n, q)) for r in range(P)]
    res = []
    try:
        for p in procs:
            p.start()
        while len(res) < P:
            try:
                res.append(q.get(timeout=600))
            except queue.Empty:
                break
            if "error" in res[-1]:
                break
    finally:
        for p in procs:
            p.join(timeout=60)
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join()
    errors = [r for r in res if "error" in r]
    assert not errors, f"rank {errors[0]['rank']}:\n{errors[0]['error']}"
    assert len(res) == P
    assert len({r["digest"] for r in res}) == 1, "the loss differs between ranks"
    assert all(r["equal"] for r in res), "angle_loss_rows is not bitwise angle_loss of the gathered logits"
    print(f"angle_loss_rows P={P} N={n}: {res[0]['loss']} on every rank")
