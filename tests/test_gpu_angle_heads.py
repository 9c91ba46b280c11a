"""-m gpu: the angle heads of Alphafold2(predict_angles=True) (alphafold2.py:813-836) on af2_angle_heads.

  * kernel against fp64 on random x: its max error must be <= 2x the max error of eager fp32 nn.Linear on the same x (the
    reference's own arithmetic), per output;
  * plane wiring: inputs whose every product and partial sum is exact, so a dropped or swapped plane pair fails;
  * the reference's fixture (tests/golden/alphafold2_angles.pt): from its trunk output, and end to end in strict and bf16 mode;
  * the distance is bitwise the one without angle heads; omega is bitwise symmetric when symmetrized;
  * memory: the call allocates its outputs only; N_res 4096 (x of 2^32 elements) on sampled rows, the last 8 included."""
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from gpu_util import check, check_strict
from oracle import heads_oracle as HO

pytestmark = pytest.mark.gpu

BUCKETS = (25, 13, 25)


def _heads(d, g, scale=1.0, buckets=BUCKETS):
    """nn.Linear-like weights of the three heads (uniform +-1/sqrt(d)), biases in the same range"""
    w = {}
    for name, nb in zip(("to_prob_theta", "to_prob_phi", "to_prob_omega"), buckets):
        w[name + ".weight"] = ((torch.rand(nb, d, generator=g, device="cuda") * 2 - 1) * d ** -0.5 * scale)
        w[name + ".bias"] = ((torch.rand(nb, generator=g, device="cuda") * 2 - 1) * d ** -0.5)
    return w


def _run(w, x, sym):
    from alphafold2_b200 import ops
    pk = ops.pack_angle_heads(w["to_prob_theta.weight"], w["to_prob_theta.bias"], w["to_prob_phi.weight"], w["to_prob_phi.bias"],
                              w["to_prob_omega.weight"], w["to_prob_omega.bias"])
    return ops.angle_heads(pk, x, sym)


@pytest.mark.parametrize("sym", [False, True])
@pytest.mark.parametrize("d", [32, 128, 256])
@pytest.mark.parametrize("b", [1, 2])
@pytest.mark.parametrize("n", [20, 64, 100, 257])
def test_kernel_against_fp64(n, b, d, sym):
    from alphafold2_b200 import ops
    assert ops.angle_heads_ok(d, BUCKETS)
    g = torch.Generator(device="cuda").manual_seed(n * 7 + b * 3 + d + sym)
    x = torch.randn(b, n, n, d, device="cuda", generator=g)
    w = _heads(d, g)
    out = _run(w, x, sym)
    again = _run(w, x, sym)
    ref = HO.angle_heads({k: v.double() for k, v in w.items()}, x.double(), sym)
    eager = HO.angle_heads(w, x, sym)                    # nn.Linear in fp32 (F.linear), the reference's arithmetic
    for name, o, o2, r, e in zip(("theta", "phi", "omega"), out, again, ref, eager):
        assert o.shape == r.shape and o.dtype == torch.float32
        assert torch.equal(o, o2), f"{name}: two identical launches differ"
        err = (o.double() - r).abs().max().item()
        err_eager = (e.double() - r).abs().max().item()
        print(f"angles n{n} b{b} d{d} sym{int(sym)} {name}: max err {err:.3e}, eager fp32 {err_eager:.3e}")
        assert err <= 2 * err_eager, f"{name}: max err {err:.3e} > 2 x eager fp32's {err_eager:.3e}"
    if sym:
        assert torch.equal(out[2], out[2].transpose(1, 2)), "symmetrized omega is not bitwise symmetric"


@pytest.mark.parametrize("buckets", [(30, 10, 10), (8, 8, 32), (1, 1, 1), (20, 20, 24), (25, 13, 26)])
def test_other_bucket_splits(buckets):
    """Bucket counts are run-time arguments.  Symmetrised, omega runs on a 32-row window of the 64 weight rows that starts at
    min(8 floor((n_theta + n_phi) / 8), 32): (30, 10, 10) uses the clamped start 32, (8, 8, 32) a full window."""
    from alphafold2_b200 import ops
    assert ops.angle_heads_ok(128, buckets)
    g = torch.Generator(device="cuda").manual_seed(sum(buckets))
    x = torch.randn(2, 37, 37, 128, device="cuda", generator=g)
    w = _heads(128, g, buckets=buckets)
    for sym in (False, True):
        out = _run(w, x, sym)
        ref = HO.angle_heads({k: v.double() for k, v in w.items()}, x.double(), sym)
        eager = HO.angle_heads(w, x, sym)
        for name, o, r, e in zip(("theta", "phi", "omega"), out, ref, eager):
            err, err_e = (o.double() - r).abs().max().item(), (e.double() - r).abs().max().item()
            assert err <= 2 * err_e, f"{buckets} sym{int(sym)} {name}: max err {err:.3e} > 2 x eager fp32's {err_e:.3e}"
        if sym:
            assert torch.equal(out[2], out[2].transpose(1, 2))


@pytest.mark.parametrize("buckets", [(25, 13, 25), (30, 10, 10), (20, 3, 30), (40, 20, 5), (1, 1, 63)])
def test_shape_rule_matches_the_c_entry(buckets):
    """ops.angle_heads_ok and af2_angle_heads accept and reject the same bucket splits; (20, 3, 30) does not fit one window
    symmetrised, (40, 20, 5) and (1, 1, 63) exceed the 64 output columns"""
    from alphafold2_b200 import _lib, ops
    nt, np_, no = buckets
    x = torch.zeros(1, 9, 9, 64, device="cuda")
    planes = torch.zeros(2, 3, 64, 32, dtype=torch.bfloat16, device="cuda")
    bias = torch.zeros(64, device="cuda")
    outs = [torch.empty(1, 9, 9, nb, device="cuda") for nb in buckets]
    for sym in (0, 1):
        rc = _lib.load().af2_angle_heads(x.data_ptr(), planes.data_ptr(), bias.data_ptr(), *(o.data_ptr() for o in outs), 1, 9, 64,
                                         nt, np_, no, sym, ops._stream_ptr())
        want = ops.angle_heads_ok(64, buckets) or (not sym and nt + np_ + no <= 64)
        assert (rc == 0) == want, f"{buckets} sym{sym}: rc {rc}, {_lib.load().af2_last_error()}"
    torch.cuda.synchronize()


def test_stores_stay_inside_the_outputs():
    """Outputs carved from NaN-filled buffers with guard regions before and after each: every output element is written, no
    guard element is (ragged n: a partial last tile in both directions; two batch elements; both omega modes)."""
    from alphafold2_b200 import _lib, ops
    G = 4096
    B, n, d = 2, 19, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, n, n, d, device="cuda", generator=g)
    w = _heads(d, g)
    pk = ops.pack_angle_heads(w["to_prob_theta.weight"], w["to_prob_theta.bias"], w["to_prob_phi.weight"], w["to_prob_phi.bias"],
                              w["to_prob_omega.weight"], w["to_prob_omega.bias"])
    for sym in (0, 1):
        bufs = [torch.full((2 * G + B * n * n * nb,), float("nan"), device="cuda") for nb in BUCKETS]
        outs = [b_[G:G + B * n * n * nb] for b_, nb in zip(bufs, BUCKETS)]
        _lib.check(_lib.load().af2_angle_heads(x.data_ptr(), pk.tensors["planes"].data_ptr(), pk.tensors["bias"].data_ptr(),
                                               *(o.data_ptr() for o in outs), B, n, d, *BUCKETS, sym, ops._stream_ptr()))
        torch.cuda.synchronize()
        for name, b_, o in zip(("theta", "phi", "omega"), bufs, outs):
            assert torch.isnan(b_[:G]).all() and torch.isnan(b_[-G:]).all(), f"sym{sym} {name}: a guard element was written"
            assert torch.isfinite(o).all(), f"sym{sym} {name}: {int((~torch.isfinite(o)).sum())} output elements not written"


def _full_mantissa(shape, g):
    m = 1.0 + torch.randint(1, 1 << 23, shape, device="cuda", generator=g).double() / (1 << 23)
    m = m + (m * (1 << 23)).remainder(2).eq(0).double() * 2.0 ** -23      # odd last bit: all 24 bits in use
    s = torch.where(torch.rand(shape, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    return (s * m * torch.exp2(torch.randint(-8, 9, shape, device="cuda", generator=g).double())).float()


def _one_hot(rows, K, g):
    idx = torch.randint(0, K, (rows,), device="cuda", generator=g)
    val = torch.exp2(torch.randint(-20, 21, (rows,), device="cuda", generator=g).float())
    val = torch.where(torch.rand(rows, device="cuda", generator=g) < 0.5, -val, val)
    v = torch.zeros(rows, K, device="cuda")
    v[torch.arange(rows, device="cuda"), idx] = val
    return v


@pytest.mark.parametrize("sym", [False, True])
@pytest.mark.parametrize("d", [32, 96, 256])
def test_plane_wiring_exact(d, sym):
    """Every output is one product: x with all 24 mantissa bits against one-hot +-2^s weight rows (passes (2,0) (1,0) (0,0) carry
    x's planes), then one-hot x against full-mantissa weights (passes (0,2) (0,1) (0,0)).  x is symmetric in (i, j), so s = x.
    Every partial sum is an fp32 value: the result must be exact, and a dropped or swapped plane pair changes it."""
    g = torch.Generator(device="cuda").manual_seed(d + 5 * sym)
    b, n = 2, 37
    for case in ("onehot_w", "onehot_x"):
        if case == "onehot_w":
            x = _full_mantissa((b, n, n, d), g)
            ws = [_one_hot(nb, d, g) for nb in BUCKETS]
        else:
            x = _one_hot(b * n * n, d, g).reshape(b, n, n, d)
            ws = [_full_mantissa((nb, d), g) for nb in BUCKETS]
        x = torch.where(torch.ones(n, n, device="cuda", dtype=torch.bool).triu()[None, :, :, None], x, x.transpose(1, 2)).contiguous()
        w = {}
        for name, wt in zip(("to_prob_theta", "to_prob_phi", "to_prob_omega"), ws):
            w[name + ".weight"], w[name + ".bias"] = wt, torch.zeros(wt.shape[0], device="cuda")
        out = _run(w, x, sym)
        ref = HO.angle_heads({k: v.double() for k, v in w.items()}, x.double(), sym)
        for name, o, r in zip(("theta", "phi", "omega"), out, ref):
            assert torch.equal(r.float().double(), r), "reference not exact in fp32"
            bad = o.double() != r
            assert not bad.any(), f"{case}/d{d}/sym{int(sym)}/{name}: {int(bad.sum())} outputs differ, first {o.double()[bad][0].item()!r} vs {r[bad][0].item()!r}"


def _model(fx, predict_angles=True, sym=False, precision=None):
    import alphafold2_b200 as A
    cfg = dict(fx["cfg"])
    cfg["predict_angles"] = predict_angles
    model = A.Alphafold2(**cfg)
    st = {k: v for k, v in fx["state"].items() if predict_angles or not k.startswith("to_prob_")}
    res = model.load_state_dict(st, strict=False)
    assert not res.unexpected_keys
    model.symmetrize_omega = sym
    if precision:
        A.set_precision(model, precision)
    return model.cuda().eval()


def _forward(model, fx):
    i = fx["inputs"]
    return model(i["seq"].cuda(), i["msa"].cuda(), mask=i["mask"].cuda(), msa_mask=i["msa_mask"].cuda())


OUTS = (("theta", "theta_logits"), ("phi", "phi_logits"), ("omega", "omega_logits"))


def _outs(fx, call, kind="out_fp64"):
    """the call's outputs: distance, theta and phi are stored once (symmetrize_omega does not change them), omega per call"""
    return {**fx[kind], **fx["calls"][call][kind]}


@pytest.mark.parametrize("call", ["sym0", "sym1"])
def test_fixture_from_trunk_output(call):
    fx = load_golden("alphafold2_angles")
    c = fx["calls"][call]
    w = {k: v.float().cuda() for k, v in fx["state"].items() if k.startswith("to_prob_")}
    out = _run(w, fx["x_fp64"].cuda(), c["symmetrize_omega"])
    for (name, key), o in zip(OUTS, out):
        check_strict(f"angles/golden/{call}/from_x/{name}", o, _outs(fx, call)[key])


@pytest.mark.parametrize("call", ["sym0", "sym1"])
def test_fixture_end_to_end(call):
    fx = load_golden("alphafold2_angles")
    c = fx["calls"][call]
    sym = c["symmetrize_omega"]
    ret = _forward(_model(fx, sym=sym, precision="strict"), fx)
    ref, ac = _outs(fx, call), _outs(fx, call, "out_autocast_bf16")
    check_strict(f"strict/angles/golden/{call}/distance", ret.distance, ref["distance"])
    for name, key in OUTS:
        check_strict(f"strict/angles/golden/{call}/{name}", getattr(ret, key), ref[key])
    ret = _forward(_model(fx, sym=sym), fx)
    for name, key in (("distance", "distance"),) + OUTS:
        check(f"angles/golden/{call}/{name}", getattr(ret, key), ref[key], ac[key].float())
    if sym:
        assert torch.equal(ret.omega_logits, ret.omega_logits.transpose(1, 2))


@pytest.mark.parametrize("precision", ["bf16", "strict"])
def test_distance_unchanged_by_angle_heads(precision):
    fx = load_golden("alphafold2_angles")
    base = _forward(_model(fx, predict_angles=False, precision=precision), fx).distance
    for sym in (False, True):
        ret = _forward(_model(fx, sym=sym, precision=precision), fx)
        assert torch.equal(ret.distance, base), f"distance changed with predict_angles (symmetrize_omega={sym})"
        assert ret.theta_logits is not None and ret.omega_logits is not None


@pytest.mark.parametrize("sym", [False, True])
def test_no_pair_sized_temporary(sym):
    """N 1024, d 256: the call allocates its three outputs and nothing of x's size (1.07 GB)"""
    N, d = 1024, 256
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(1, N, N, d, device="cuda", generator=g)
    w = _heads(d, g)
    _run(w, x[:, :8, :8].contiguous(), sym)                 # packing and module load outside the measured call
    from alphafold2_b200 import ops
    pk = ops.pack_angle_heads(w["to_prob_theta.weight"], w["to_prob_theta.bias"], w["to_prob_phi.weight"], w["to_prob_phi.bias"],
                              w["to_prob_omega.weight"], w["to_prob_omega.bias"])
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = ops.angle_heads(pk, x, sym)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    outputs = sum(o.numel() * 4 for o in out)
    print(f"angle heads N{N} sym{int(sym)}: peak +{extra / 1e6:.1f} MB, outputs {outputs / 1e6:.1f} MB, x {x.numel() * 4 / 1e6:.0f} MB")
    assert extra <= outputs + (8 << 20), f"allocated {extra} B beyond its {outputs} B of outputs"


N_BIG = 4096
ROWS = [0, 1, 1000, 2047, 2048, 3001] + list(range(N_BIG - 8, N_BIG))


def test_n4096_rows_against_eager():
    """x of exactly 2^32 elements: 64-bit token offsets.  Sampled rows against eager fp32 and fp64 on those rows."""
    N, d = N_BIG, 256
    assert N * N * d == 2 ** 32
    free, _ = torch.cuda.mem_get_info()
    if free < 26e9:
        pytest.skip(f"needs 26 GB free, {free / 1e9:.1f} GB")
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(1, N, N, d, device="cuda", generator=g)
    w = _heads(d, g)
    w64 = {k: v.double() for k, v in w.items()}
    rows = torch.tensor(ROWS, device="cuda")
    xr = x[0, rows]                                            # [r, N, d]: pairs (row, j)
    xt = x[0, :, rows].transpose(0, 1)                         # [r, N, d]: pairs (j, row)
    for sym in (False, True):
        theta, phi, omega = _run(w, x, sym)
        got = (theta[0, rows], phi[0, rows], omega[0, rows])
        s32 = (xr + xt) * 0.5 if sym else xr
        s64 = (xr.double() + xt.double()) * 0.5 if sym else xr.double()
        eager = (F.linear(xr, w["to_prob_theta.weight"], w["to_prob_theta.bias"]), F.linear(xr, w["to_prob_phi.weight"], w["to_prob_phi.bias"]),
                 F.linear(s32, w["to_prob_omega.weight"], w["to_prob_omega.bias"]))
        ref = (HO._lin(w64, "to_prob_theta", xr.double()), HO._lin(w64, "to_prob_phi", xr.double()), HO._lin(w64, "to_prob_omega", s64))
        for name, o, e, r in zip(("theta", "phi", "omega"), got, eager, ref):
            err, err_e = (o.double() - r).abs().max().item(), (e.double() - r).abs().max().item()
            print(f"N4096 sym{int(sym)} {name}: max err {err:.3e}, eager fp32 {err_e:.3e} on rows {ROWS}")
            assert err <= 2 * err_e, f"sym{int(sym)}/{name}: max err {err:.3e} > 2 x eager fp32's {err_e:.3e}"
        if sym:
            assert torch.equal(omega[0, rows], omega[0, :, rows].transpose(0, 1)), "omega not symmetric on the sampled rows"
        del theta, phi, omega
