"""-m gpu: the structure module under parallel.shard_alphafold2(pair_rows=True), with P ranks on ONE GPU (the harness of
tests/test_gpu_sharded_pair_rows.py: P processes on cuda:0 in a gloo group, collectives staged through host memory), at P = 2, 3
and 4, even and uneven N_res, structure heads 1 and 4, structure depth 0 and 2, on an Alphafold2 with templates, template angles,
an extra MSA, recyclables and the angle heads.  Gates, on every rank, against the default shard_alphafold2 forward:
  * coords and confidence bitwise equal (whole on every rank); the distogram and angle rows bitwise those rows;
  * ret.recyclables: coords and single_msa_repr_row bitwise, pairwise_repr [1, n1 - n0, N, d] and bitwise those rows;
  * a second iteration fed the rank's own row recyclables, and one fed the default's whole recyclables, give coordinates and
    distance rows bitwise those of the default's second iteration;
  * every return-flag combination returns what Alphafold2.forward returns (types, keys and shapes; rows where they are rows);
  * peak allocated memory: with coordinates at most the pair projection's scratch band, its GEMM workspace, the structure
    layer's workspace, the per-residue buffers and 2 MiB above the same forward with return_trunk=True, and at least
    (1 - 1/P) 4 N^2 d below the default mode with coordinates;
and on rank 0: the coordinates and the gathered distogram of a forward without templates or extra MSA against the fp64 oracle.
Not covered here: the peer-store exchange, NCCL and graph replay (they need one GPU per rank)."""
import itertools
import os

import pytest
import torch

import test_gpu_sharded_model_ranks as H
import test_gpu_sharded_pair_rows as PR

pytestmark = pytest.mark.gpu

# P, n, S, T, structure heads, structure depth   (d = 128: the distogram head kernel's smallest dim)
CASES = [
    (2, 40, 4, 1, 1, 2),       # even
    (3, 43, 5, 2, 4, 2),       # pair shards 15/14/14
    (4, 48, 4, 1, 4, 0),       # even, no structure layer
    (4, 50, 5, 2, 1, 2),       # pair shards 13/13/12/12
]
D = 128
FLAGS = list(itertools.product((False, True), repeat=3))       # return_confidence, return_recyclables, return_aux_logits


def _flat(out):
    """A forward's return value as {name: tensor}, in the shape Alphafold2.forward gives it."""
    if torch.is_tensor(out):
        return {"coords": out}
    coords, second = out
    if torch.is_tensor(second):
        return {"coords": coords, "confidence": second}
    res = {"coords": coords, "distance": second.distance, "theta": second.theta_logits, "phi": second.phi_logits,
           "omega": second.omega_logits}
    if second.recyclables is not None:
        r = second.recyclables
        res.update(rec_coords=r.coords, rec_single=r.single_msa_repr_row, rec_pair=r.pairwise_repr)
    return res


ROWS = ("distance", "theta", "phi", "omega", "rec_pair")       # this rank's pair rows in the rows mode


def _same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _compare(rows, default, n0, n1):
    """Names whose rows-mode value is not bitwise the default's (its rows [n0, n1) for the pair-row outputs)."""
    bad = sorted(set(rows) ^ set(default))
    for k in set(rows) & set(default):
        want = default[k][:, n0:n1] if k in ROWS else default[k]
        if not _same(rows[k].cpu(), want.cpu()):
            bad.append(k)
    return bad


def _stage_broadcast_through_host():
    import torch.distributed as dist
    broadcast = dist.broadcast

    def staged(t, src=None, group=None, async_op=False, group_src=None):
        assert not async_op
        host = t.detach().contiguous().cpu()
        broadcast(host, src=src, group=group, group_src=group_src)
        t.copy_(host)

    dist.broadcast = staged


def _run(rank, P, case):
    import torch.distributed as dist
    import alphafold2_b200 as A
    from alphafold2_b200 import ops, parallel
    from gpu_util import check, depth_gates, to64
    from oracle import evoformer_oracle as O
    from oracle import structure_oracle as SO
    n, S, T, heads, depth = case
    torch.manual_seed(0)
    model = A.attach_structure_module(A.Alphafold2(dim=D, depth=2, heads=2, dim_head=32, max_seq_len=n, extra_msa_evoformer_layers=1,
                                                   templates_embed_layers=1, predict_angles=True, predict_coords=True,
                                                   structure_module_depth=depth, structure_module_heads=heads))
    st = O.randomize_zero_init_({k: v.clone() for k, v in model.state_dict().items()}, std=0.05)
    model.load_state_dict(st)
    model = model.cuda().eval()
    seq, mask, kw = H._model_inputs(D, n, S, T)
    on = parallel.shard_offsets(n, P)
    n0, n1 = on[rank], on[rank + 1]
    fwd = lambda **f: model(seq, mask=mask, **{**kw, **f})  # noqa: E731
    res = {}

    parallel.shard_alphafold2(model, use_graph=False)
    default = {f: _flat(fwd(return_confidence=f[0], return_recyclables=f[1], return_aux_logits=f[2])) for f in FLAGS}
    rec_whole = A.Recyclables(default[FLAGS[-1]]["rec_coords"], default[FLAGS[-1]]["rec_single"], default[FLAGS[-1]]["rec_pair"])
    second = _flat(fwd(recyclables=rec_whole, return_aux_logits=True))
    _, mem_default = PR._peak(lambda: fwd(return_confidence=True))

    parallel.shard_alphafold2(model, use_graph=False, pair_rows=True)
    rows = {f: _flat(fwd(return_confidence=f[0], return_recyclables=f[1], return_aux_logits=f[2])) for f in FLAGS}
    res["flags_bad"] = {f: bad for f in FLAGS if (bad := _compare(rows[f], default[f], n0, n1))}
    rec_rows = A.Recyclables(rows[FLAGS[-1]]["rec_coords"], rows[FLAGS[-1]]["rec_single"], rows[FLAGS[-1]]["rec_pair"])
    res["rec_pair_shape"] = tuple(rec_rows.pairwise_repr.shape) == (1, n1 - n0, n, D)
    keep = ("coords", "distance")
    second_default = {k: second[k] for k in keep}
    res["second_own_rows_bad"] = _compare({k: v for k, v in _flat(fwd(recyclables=rec_rows, return_aux_logits=True)).items()
                                           if k in keep}, second_default, n0, n1)
    res["second_whole_bad"] = _compare({k: v for k, v in _flat(fwd(recyclables=rec_whole, return_aux_logits=True)).items()
                                        if k in keep}, second_default, n0, n1)
    del rows, default, second, rec_rows, rec_whole

    peaks = {}
    for name, f in (("trunk", dict(return_trunk=True)), ("coords", dict(return_confidence=True))) * 2:
        _, peaks[name] = PR._peak(lambda: fwd(**f))
    R = n1 - n0
    lib = ops._lib.load()
    band = ops.plan_pair_projection_band(R, n, D, "bf16", 1 << 40)
    res["allowance"] = (band * n * D * 4 + lib.af2_template_embed_workspace(band * n, D) + lib.af2_structure_layer_rows_workspace(n, R, D, heads)
                        + n * (4 + 3 + 9 + 3 + 1 + 2 * D) * 4 + (2 << 20))
    res["mem"] = (mem_default, peaks["trunk"], peaks["coords"])
    res["pair_bytes"] = 4 * n * n * D

    # the fp64 oracle covers the trunk with recyclables and the structure module (no templates, no extra MSA)
    rc = kw["recyclables"]
    coords, ret = model(seq, kw["msa"], mask=mask, msa_mask=kw["msa_mask"], recyclables=rc, return_aux_logits=True)
    distance = parallel.gather_pair_rows(ret.distance)
    if rank == 0:
        w = {k: v.cuda() for k, v in to64(st).items()}
        rec = A.Recyclables(rc.coords.double(), rc.single_msa_repr_row.double(), rc.pairwise_repr.double())
        ref = SO.alphafold2_coords(w, seq, kw["msa"], mask, kw["msa_mask"], 2, 2, heads, depth, recyclables=rec, dtype=torch.float64)
        gates = depth_gates(2 + depth)
        tag = f"sharded_structure_rows_p{P}_one_gpu/n{n}h{heads}depth{depth}"
        res["vs_oracle"] = (check(f"{tag}/coords", coords, ref["coords"], **gates)["max_rel"],
                            check(f"{tag}/distance", distance, ref["distance"], **gates)["max_rel"])
    dist.barrier()
    return res


def _worker(rank, P, port, case, q):
    import datetime
    import sys
    import traceback
    import torch.distributed as dist
    sys.path[:0] = [H.ROOT, os.path.join(H.ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    res = {"rank": rank}
    try:
        from test_gpu_sharded_ranks_uneven import _stage_collectives_through_host
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=300))
        try:
            _stage_collectives_through_host()
            _stage_broadcast_through_host()
            with torch.no_grad():
                res.update(_run(rank, P, case))
        finally:
            dist.destroy_process_group()
    except BaseException:  # noqa: BLE001 - reported to the parent, which fails the test with it
        res["error"] = traceback.format_exc()
    q.put(res)


def _spawn(P, case):
    import queue
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
    procs = [ctx.Process(target=_worker, args=(r, P, port, case, q)) for r in range(P)]
    res = []
    try:
        for p in procs:
            p.start()
        while len(res) < P:
            try:
                res.append(q.get(timeout=900))
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
    assert len(res) == P, f"{P - len(res)} of {P} ranks did not report within the timeout"
    return sorted(res, key=lambda r: r["rank"])


@pytest.mark.parametrize("P,n,S,T,heads,depth", CASES)
def test_structure_module_pair_rows_one_gpu(P, n, S, T, heads, depth):
    res = _spawn(P, (n, S, T, heads, depth))
    for r in res:
        mem_default, mem_trunk, mem_coords = r["mem"]
        print(f"  rank {r['rank']}: peak allocated {mem_coords / 2**20:.2f} MiB rows with coordinates, {mem_trunk / 2**20:.2f} MiB "
              f"rows return_trunk, {mem_default / 2**20:.2f} MiB default with coordinates (one fp32 pair tensor "
              f"{r['pair_bytes'] / 2**20:.2f} MiB, allowance {r['allowance'] / 2**20:.2f} MiB; P={P} processes on one GPU)")
        assert not r["flags_bad"], (r["rank"], r["flags_bad"])
        assert r["rec_pair_shape"], r["rank"]
        assert not r["second_own_rows_bad"], (r["rank"], r["second_own_rows_bad"])
        assert not r["second_whole_bad"], (r["rank"], r["second_whole_bad"])
        assert mem_coords - mem_trunk <= r["allowance"], (r["rank"], r["mem"], r["allowance"])
        assert mem_default - mem_coords >= (1 - 1 / P) * r["pair_bytes"], (r["rank"], r["mem"], r["pair_bytes"])
    print(f"structure rows P={P} n={n} heads={heads} depth={depth}: coords / distance vs fp64 max_rel {res[0]['vs_oracle']}")
