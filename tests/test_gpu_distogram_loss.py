"""-m gpu: the distogram loss (utils.distogram_loss, utils.get_bucketed_distance_matrix, parallel.distogram_loss_rows) against
the reference's outputs in tests/golden/distogram_loss.pt and the fp64 oracle (oracle/distogram_loss_oracle.py).

  * labels bitwise the fixture and the oracle: N past 25, distances on the edges, NaN coordinates, nb 1 / 2 / 37 / 64, [N, c]
    input, c 1 / 3 / 4;
  * the loss within oracle.loss_bound of the fp64 loss (the bound is derived from the kernel's rounding points; its CPU
    controls are in tests/test_oracle_distogram_loss.py) and within fp32 rounding of the reference's value;
  * the quirks: an in-range ignore_index, an all-masked batch (NaN), mask=None, a batch mean across elements;
  * the contract: reproducible bits, two launches and no host synchronisation, 16 bytes per (element, row) above the inputs,
    a shape past 2^31 logits elements, and refusals before any launch;
  * per-row partials of any split of the rows combine bitwise to the whole; and parallel.distogram_loss_rows on the rows of a
    shard_alphafold2(pair_rows=True) forward at P = 2, 3 and 4 on one GPU (the harness of tests/test_gpu_sharded_model_ranks.py)
    returns on every rank bitwise utils.distogram_loss of the gathered distogram."""
import os
import queue

import pytest
import torch

from oracle import distogram_loss_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["small", "small_ignore3", "edges16", "masked", "large", "large16"]


def _u():
    from alphafold2_b200 import utils
    return utils


def _launches():
    from alphafold2_b200 import _lib
    return _lib.load().af2_launch_count()


@pytest.fixture(scope="module")
def fx(golden):
    return golden("distogram_loss")


def _check_loss(got, logits, lab, ii, ref=None):
    want = O.loss64(logits.cpu(), lab.cpu(), ii).item()
    bound = O.loss_bound(logits.cpu(), lab.cpu(), ii)
    err = abs(got.item() - want)
    assert err <= bound, (got.item(), want, err, bound)
    if ref is not None:
        assert abs(got.item() - ref) <= 64 * 2 ** -24 * abs(ref) + bound, (got.item(), ref)
    return err / bound if bound else 0.0


@pytest.mark.parametrize("name", CASES)
def test_fixture(fx, name):
    U = _u()
    c = fx[name]
    x, m, lg = c["coords"].cuda(), c["mask"].cuda(), c["logits"].cuda()
    lab = U.get_bucketed_distance_matrix(x, m, c["nb"], c["ignore_index"])
    assert lab.dtype == torch.int64 and torch.equal(lab.cpu(), c["labels"])
    loss = U.distogram_loss(lg, x, m, c["ignore_index"])
    assert loss.dim() == 0 and loss.dtype == torch.float32 and loss.is_cuda
    _check_loss(loss, lg, c["labels"], c["ignore_index"], ref=c["loss"].item())


def _coords(b, n, c, g, scale=8.0, nan=False, edges=False):
    x = torch.randn(b, n, c, generator=g) * scale + 20.0
    if edges:                          # residues on a line 0.5 A apart: many distances exactly on the nb 37 edges
        x[0, : min(n, 40)] = 0.0
        x[0, : min(n, 40), 0] = torch.arange(min(n, 40), dtype=torch.float32) * 0.5
    if nan:
        x[-1, n // 3, 0] = float("nan")
    return x


@pytest.mark.parametrize("b,n,c,nb", [(2, 100, 3, 37), (1, 257, 3, 1), (3, 64, 3, 2), (2, 130, 3, 64), (1, 90, 1, 37),
                                      (2, 75, 4, 37), (1, 333, 3, 16)])
def test_labels_vs_oracle(b, n, c, nb):
    U = _u()
    g = torch.Generator().manual_seed(n + nb)
    x = _coords(b, n, c, g, nan=True, edges=c == 3)
    mask = torch.rand(b, n, generator=g) > 0.2
    lab = U.get_bucketed_distance_matrix(x.cuda(), mask.cuda(), nb, -7)
    want = O.labels(x, mask, nb, -7)
    assert torch.equal(lab.cpu(), want)
    if nb > 1:
        assert (want == nb - 1).any() and (want == 0).any()
    flat = U.get_bucketed_distance_matrix(x[0].cuda(), mask[0].cuda(), nb, -7)
    assert flat.shape == (n, n) and torch.equal(flat.cpu(), want[0])
    assert torch.equal(U.get_bucketed_distance_matrix(x.cuda(), None, nb).cpu(), O.labels(x, None, nb))


@pytest.mark.parametrize("b,n,nb,scale", [(1, 300, 37, 3.0), (2, 129, 37, 30.0), (3, 64, 64, 3.0), (1, 77, 2, 3.0), (2, 40, 1, 3.0),
                                          (1, 50, 200, 2.0), (16, 40, 37, 3.0)])
def test_loss_vs_oracle(b, n, nb, scale):
    U = _u()
    g = torch.Generator().manual_seed(b * 1000 + n)
    x = _coords(b, n, 3, g, nan=True, edges=True)
    mask = torch.rand(b, n, generator=g) > 0.15
    lg = torch.randn(b, n, n, nb, generator=g) * scale
    loss = U.distogram_loss(lg.cuda(), x.cuda(), mask.cuda())
    _check_loss(loss, lg, O.labels(x, mask, nb), -100)


def test_quirks():
    U = _u()
    g = torch.Generator().manual_seed(9)
    b, n, nb = 3, 50, 37
    x, lg = _coords(b, n, 3, g), torch.randn(b, n, n, nb, generator=g)
    mask = torch.ones(b, n, dtype=torch.bool)
    mask[0, :30] = False                                            # elements of different mask counts
    mask[1, 5:] = False
    xc, lc, mc = x.cuda(), lg.cuda(), mask.cuda()
    for ii in (3, 36, 0, -100, 1000):                               # in range: the bucket drops out too
        lab = O.labels(x, mask, nb, ii)
        _check_loss(U.distogram_loss(lc, xc, mc, ii), lg, lab, ii)
    lab = O.labels(x, mask, nb)
    # the batch mean runs over the counted pairs, not the mean of per-element means
    t = O.terms64(lg, lab, -100)
    assert abs(t.mean().item() - U.distogram_loss(lc, xc, mc).item()) <= O.loss_bound(lg, lab)
    _check_loss(U.distogram_loss(lc, xc), lg, O.labels(x, None, nb), -100)       # mask=None
    assert torch.isnan(U.distogram_loss(lc, xc, torch.zeros_like(mc)))            # nothing counts: 0 / 0
    assert torch.equal(U.distogram_loss(lc, xc, None), U.distogram_loss(lc, xc, torch.ones_like(mc)))


def test_contract_bits_launches_memory():
    U = _u()
    g = torch.Generator().manual_seed(4)
    b, n, nb = 2, 1000, 37
    x = (torch.randn(b, n, 3, generator=g) * 10).cuda()
    lg = torch.randn(b, n, n, nb, generator=g).cuda()
    mask = (torch.rand(b, n, generator=g) > 0.1).cuda()
    U.distogram_loss(lg, x, mask)                                   # the bucket edges are cached on first use
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    k0 = _launches()
    first = U.distogram_loss(lg, x, mask)
    assert _launches() - k0 == 2
    second = U.distogram_loss(lg, x, mask)
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int32), second.view(torch.int32))
    assert torch.cuda.max_memory_allocated() - base <= 16 * b * n + 4096
    # no host synchronisation: the calls enqueue behind a long kernel and return before it ends
    torch.cuda._sleep(200_000_000)
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    U.distogram_loss(lg, x, mask)
    assert not start.query(), "distogram_loss waited for the device"
    torch.cuda.synchronize()


def test_past_2_31_elements():
    U = _u()
    n, nb = 7700, 37
    assert n * n * nb > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(1)
    lg = torch.randn(1, n, n, nb, device="cuda", generator=g)
    x = torch.randn(1, n, 3, device="cuda", generator=g) * 15
    mask = torch.ones(1, n, dtype=torch.bool, device="cuda")
    mask[0, -7:] = False
    loss = U.distogram_loss(lg, x, mask)
    lab = O.labels(x.cpu(), mask.cpu(), nb)
    want, bound, k, tail = 0.0, 0.0, 0, None
    for r0 in range(0, n, 700):                                     # the fp64 oracle in row blocks
        lab_r, lg_r = lab[:, r0:r0 + 700], lg[:, r0:r0 + 700].cpu()
        t = O.terms64(lg_r, lab_r, -100)
        want += t.sum().item()
        k += t.numel()
        bound += O.term_bound(lg_r, lab_r, -100).sum().item()
        del lg_r
    want /= k
    assert abs(loss.item() - want) <= bound / k + 2 ** -23 * abs(want) + 1e-12


def test_refusals():
    U = _u()
    x = torch.randn(1, 8, 3, device="cuda")
    lg = torch.randn(1, 8, 8, 37, device="cuda")
    m = torch.ones(1, 8, dtype=torch.bool, device="cuda")
    bad = [
        (lambda: U.distogram_loss(lg.cpu(), x, m), RuntimeError),
        (lambda: U.distogram_loss(lg, x.cpu(), m), RuntimeError),
        (lambda: U.distogram_loss(lg.clone().requires_grad_(), x, m), RuntimeError),
        (lambda: U.distogram_loss(lg, x.clone().requires_grad_(), m), RuntimeError),
        (lambda: U.distogram_loss(lg, x[:, :7], m), ValueError),
        (lambda: U.distogram_loss(lg, x.expand(2, 8, 3), m), ValueError),
        (lambda: U.distogram_loss(lg, x, m[:, :7]), ValueError),
        (lambda: U.distogram_loss(lg[:, :7], x, m), ValueError),
        (lambda: U.distogram_loss(lg[0], x, m), ValueError),
        (lambda: U.distogram_loss(lg[..., :0], x, m), ValueError),
        (lambda: U.distogram_loss(lg[:, :0, :0], x[:, :0], m[:, :0]), ValueError),
        (lambda: U.distogram_loss(lg[:0], x[:0], m[:0]), ValueError),
        (lambda: U.distogram_loss(lg, x, m, ignore_index=-100.0), TypeError),
        (lambda: U.distogram_loss(lg, x, m, ignore_index=True), TypeError),
        (lambda: U.distogram_loss(lg, x, m.float()), TypeError),
        (lambda: U.distogram_loss(lg, x[..., :0], m), ValueError),
        (lambda: U.get_bucketed_distance_matrix(x.cpu(), m.cpu()), RuntimeError),
        (lambda: U.get_bucketed_distance_matrix(x, m, 0), ValueError),
        (lambda: U.get_bucketed_distance_matrix(x, m, 37, 1.5), TypeError),
        (lambda: U.get_bucketed_distance_matrix(x, m[:, :5]), ValueError),
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
    b, nb = 2, 37
    x, lg = (torch.randn(b, n, 3, generator=g) * 8).cuda(), torch.randn(b, n, n, nb, generator=g).cuda()
    mask = (torch.rand(b, n, generator=g) > 0.2).cuda()
    whole = ops.distogram_xent_rows(lg, x, mask, -100)
    parts, r0 = [], 0
    for r in splits:
        parts.append(ops.distogram_xent_rows(lg[:, r0:r0 + r].contiguous(), x, mask, -100, row0=r0))
        r0 += r
    joined = torch.cat(parts, 1)
    assert torch.equal(joined, whole)
    assert torch.equal(ops.distogram_xent_finish(joined.contiguous()).view(torch.int32), U.distogram_loss(lg, x, mask).view(torch.int32))


# ---- sharded: parallel.distogram_loss_rows on the ranks of shard_alphafold2(pair_rows=True), P processes on cuda:0 ----
SHARD_CASES = [(2, 40), (3, 43), (4, 48), (4, 50)]


def _run_rows(rank, P, n):
    import alphafold2_b200 as A
    from alphafold2_b200 import parallel, utils
    from oracle import evoformer_oracle as E
    from test_gpu_sharded_ranks_uneven import _digest
    torch.manual_seed(0)
    d = 128
    model = A.Alphafold2(dim=d, depth=1, heads=2, dim_head=32, max_seq_len=n)
    model.load_state_dict(E.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05))
    model = model.cuda().eval()
    seq = torch.randint(0, 21, (1, n)).cuda()
    msa = torch.randint(0, 21, (1, 3, n)).cuda()
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[:, -n // 8:] = False
    mask = mask.cuda()
    coords = (torch.randn(1, n, 3) * 8).cuda()
    parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)
    with torch.no_grad():
        ret = model(seq, msa, mask=mask)
    rows_loss = parallel.distogram_loss_rows(ret.distance, coords, mask)
    rows_loss_nomask = parallel.distogram_loss_rows(ret.distance, coords, None, ignore_index=5)
    whole = parallel.gather_pair_rows(ret.distance)
    ref = utils.distogram_loss(whole, coords, mask)
    ref_nomask = utils.distogram_loss(whole, coords, None, ignore_index=5)
    return {"digest": _digest(rows_loss.cpu(), rows_loss_nomask.cpu()),
            "equal": torch.equal(rows_loss.view(torch.int32), ref.view(torch.int32))
            and torch.equal(rows_loss_nomask.view(torch.int32), ref_nomask.view(torch.int32)),
            "loss": rows_loss.item()}


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
def test_distogram_loss_rows_sharded_one_gpu(P, n):
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
    assert all(r["equal"] for r in res), "distogram_loss_rows is not bitwise distogram_loss of the gathered distogram"
    print(f"distogram_loss_rows P={P} N={n}: {res[0]['loss']:.6f} on every rank")
