"""Device time, launches, template-stack calls and peak memory of alphafold2_b200.recycle against the caller's own recycling loop
on a sharded model, one process per rank, one GPU per rank (NCCL):
   python tools/time_sharded_recycle.py [--ranks 1] [--modes evoformer default rows] [--steps 3] [--num-recycles 3]
                                        [--templates 4] [--n-res 256] [--msa-rows 128] [--depth 12]
   -> one JSON line per mode, from rank 0, with every rank's numbers

Model and inputs as tools/time_recycle_loop.py's (bench.py's C2 shape with the structure module and T templates).  Modes:
evoformer = parallel.shard_evoformer(model), default = parallel.shard_alphafold2(model), rows = shard_alphafold2(model,
pair_rows=True), all eager (use_graph=False).  The manual loop is the one of tools/time_recycle_loop.py.  Reported:
  manual_ms / recycle_ms        per prediction (num_recycles + 1 forwards), rank 0's CUDA events, median of --steps rounds taken
                                alternately after one warm-up of each, with min and max
  launches_manual / _recycle    kernels of this library per prediction, per rank
  stack_calls_manual / _recycle calls of the template pair stack per prediction, per rank (parallel.sharded_template_pair_stack,
                                or Alphafold2.template_pair_stack where the branch runs whole)
  peak_alloc_manual / _recycle  torch.cuda.max_memory_allocated over one prediction, each from a released workspace, per rank
  template_reuse                model.last_template_reuse after recycle, per rank
  outputs_equal                 coordinates and confidence bitwise equal, per rank
--ranks P > 1 needs P GPUs: the ranks run concurrently and exchange over NCCL.  With fewer GPUs the script refuses; speed
with several ranks is then not measured.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _worker(rank, P, port, args, q):
    import datetime
    import torch.distributed as dist
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=P, timeout=datetime.timedelta(seconds=600),
                            device_id=torch.device("cuda", rank))
    try:
        with torch.no_grad():
            q.put(_run(rank, P, args))
    except BaseException as ex:  # noqa: BLE001 - reported by the parent
        import traceback
        q.put({"rank": rank, "error": f"{ex!r}\n{traceback.format_exc()}"})
    finally:
        dist.destroy_process_group()


def _run(rank, P, args):
    import alphafold2_b200 as A
    from alphafold2_b200 import _lib, ops, parallel
    from bench import CFG, randomize_zero_init_
    from time_recycle_loop import _card, manual_loop
    n, S, R, T = args.n_res, args.msa_rows, args.num_recycles, args.templates
    dev = torch.device("cuda", rank)
    lib = _lib.load()
    out = {"rank": rank, "card": _card(dev) if rank == 0 else None, "modes": {}}
    for mode in args.modes:
        cfg = dict(CFG, depth=args.depth)
        torch.manual_seed(0)
        model = A.attach_structure_module(A.Alphafold2(**cfg, max_seq_len=max(n, 2048), predict_coords=True))
        randomize_zero_init_(model)
        model = model.to(dev).eval()
        seq = torch.randint(0, 21, (1, n), device=dev)
        msa = torch.randint(0, 21, (1, S, n), device=dev)
        g = torch.Generator(device=dev).manual_seed(5)
        kw = dict(mask=torch.ones(1, n, dtype=torch.bool, device=dev), msa_mask=torch.ones(1, S, n, dtype=torch.bool, device=dev),
                  templates_feats=torch.randn(1, T, n, n, model.to_template_embed.in_features, device=dev, generator=g),
                  templates_angles=torch.randn(1, T, n, model.template_angle_mlp[0].in_features, device=dev, generator=g),
                  templates_mask=torch.ones(1, T, n, dtype=torch.bool, device=dev))
        if mode == "evoformer":
            parallel.shard_evoformer(model, use_graph=False)
            owner, name = model, "template_pair_stack"
        else:
            parallel.shard_alphafold2(model, use_graph=False, pair_rows=mode == "rows")
            owner, name = parallel, "sharded_template_pair_stack"
        fn, calls = getattr(owner, name), [0]

        def counted(*a, **k):
            calls[0] += 1
            return fn(*a, **k)

        setattr(owner, name, counted)
        runs = {"manual": lambda: manual_loop(model, seq, msa, R, **kw),
                "recycle": lambda: A.recycle(model, seq, msa, num_recycles=R, return_confidence=True, **kw)}
        res, outs = {}, {}
        for which in ("manual", "recycle"):
            ops.release_workspace(dev)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(dev)
            calls[0], l0 = 0, lib.af2_launch_count()
            outs[which] = tuple(t.cpu() for t in runs[which]())
            torch.cuda.synchronize()
            res[f"peak_alloc_{which}_bytes"] = torch.cuda.max_memory_allocated(dev)
            res[f"launches_{which}"] = int(lib.af2_launch_count() - l0)
            res[f"stack_calls_{which}"] = calls[0]
        res["outputs_equal"] = all(torch.equal(a, b) for a, b in zip(outs["manual"], outs["recycle"]))
        res["template_reuse"] = getattr(model, "last_template_reuse", None)
        times = {"manual": [], "recycle": []}
        for rnd in range(args.steps + 1):
            for which in ("manual", "recycle"):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                runs[which]()
                b.record()
                b.synchronize()
                if rnd > 0:
                    times[which].append(a.elapsed_time(b))
        for which, ts in times.items():
            res[f"{which}_ms"] = statistics.median(ts)
            res[f"{which}_ms_min_max"] = [min(ts), max(ts)]
        setattr(owner, name, fn)
        out["modes"][mode] = res
        del model, runs, outs
        ops.release_workspace(dev)
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=1)
    ap.add_argument("--modes", nargs="+", default=["evoformer", "default", "rows"], choices=["evoformer", "default", "rows"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--num-recycles", type=int, default=3)
    ap.add_argument("--templates", type=int, default=4)
    ap.add_argument("--n-res", type=int, default=256)
    ap.add_argument("--msa-rows", type=int, default=128)
    ap.add_argument("--depth", type=int, default=12)
    args = ap.parse_args()
    P = args.ranks
    if args.templates < 1 or args.num_recycles < 1 or args.steps < 1:
        raise SystemExit("--templates, --num-recycles and --steps must be at least 1")
    if torch.cuda.device_count() < P:
        raise SystemExit(f"--ranks {P} needs {P} GPUs (one per rank), {torch.cuda.device_count()} visible: not measured")
    import queue
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, P, port, args, q)) for r in range(P)]
    for p in procs:
        p.start()
    res = []
    try:
        while len(res) < P:
            res.append(q.get(timeout=3600))
            if "error" in res[-1]:
                break
    except queue.Empty:
        pass
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.terminate()
                p.join()
    errors = [r for r in res if "error" in r]
    if errors or len(res) < P:
        raise SystemExit(f"rank failed: {errors[0] if errors else f'{P - len(res)} ranks did not report'}")
    res.sort(key=lambda r: r["rank"])
    card = res[0]["card"]
    per_rank = ("peak_alloc_manual_bytes", "peak_alloc_recycle_bytes", "launches_manual", "launches_recycle", "stack_calls_manual",
                "stack_calls_recycle", "template_reuse", "outputs_equal")
    for mode in args.modes:
        r0 = res[0]["modes"][mode]
        line = {"mode": mode, "ranks": P, "T": args.templates, "num_recycles": args.num_recycles, "steps": args.steps,
                "what": f"C2-shaped Alphafold2(depth={args.depth}, predict_coords=True) N_res={args.n_res} MSA={args.msa_rows} "
                        f"batch=1, {args.templates} templates, eager; ms per prediction on rank 0, CUDA events",
                "manual_ms": r0["manual_ms"], "recycle_ms": r0["recycle_ms"], "manual_ms_min_max": r0["manual_ms_min_max"],
                "recycle_ms_min_max": r0["recycle_ms_min_max"], "saving": 1 - r0["recycle_ms"] / r0["manual_ms"]}
        line.update({k: [r["modes"][mode][k] for r in res] for k in per_rank})
        print(json.dumps(dict(line, **card)), flush=True)


if __name__ == "__main__":
    main()
