"""-m gpu: the GEMM epilogue through shared memory and TMA stores (gemm_tc.cuh), element-wise against fp64.

launch_gemm sends a BN = 256 epilogue kind through TMA when the call's output (and residual) have 16-byte aligned bases and
pitches and, channel-major, cm_inner is a multiple of 64 that divides M; otherwise it stores from registers.  The cases
of test_gpu_kernels.py mostly use pitches TMA cannot express, so here the same checks (fp64 bound on every element, NaN
everywhere outside the output) run on layouts on each side of that choice: "tma" is aligned, "edge" misses it by one
condition: token-major rows that end inside a 16-byte segment (odd column count, aligned pitch), or channel-major M not a
multiple of cm_inner.
"""
import pytest
import torch

import test_gpu_kernels as tk

pytestmark = pytest.mark.gpu

BN256_KINDS = ["store_tok", "store_tok_sig", "store_ch", "store_ch_rs", "gated_tok_gelu", "gated_ch_sig", "gated_ch_sig_rs",
               "resid_f32", "store_f32"]


def _out_index(batch, M, ncols, layout, store, dev, f32):
    b = torch.arange(batch, device=dev)[:, None, None]
    r = torch.arange(M, device=dev)[None, :, None]
    c = torch.arange(ncols, device=dev)[None, None, :]
    epe = 4 if f32 else 8                                      # elements per 16 bytes
    off = 0
    if layout == 0:
        ld = (ncols + epe - 1) // epe * epe + epe
        ob = M * ld + epe
        idx = off + b * ob + r * ld + c
        kw = dict(ld_out=ld, out_batch=ob)
    else:
        inner, pitch = 64, 72
        ld = (M + inner - 1) // inner * pitch + 8
        ob = ld * ncols + 8
        idx = off + b * ob + c * ld + (r // inner) * pitch + r % inner
        kw = dict(ld_out=ld, out_batch=ob, cm_inner=inner, cm_pitch=pitch)
    size = off + batch * kw["out_batch"] + 16
    return idx, size, off, kw


def _run(monkeypatch, kind, store, M, K, batch, seed, mn_major=False, nout=None):
    mode, act, layout, rs = tk.KINDS[kind]
    f32 = mode in (2, 3)
    W = 128 if mode == 1 else 256
    if nout is None:
        nout = W + W // 2 + (1 if store == "edge" and layout == 0 else 8)   # partial last column tile
    if layout == 1 and store == "edge":
        M += 8
    monkeypatch.setattr(tk, "_out_index", lambda bt, m, n, lay, st, dev: _out_index(bt, m, n, lay, st, dev, f32))
    batch = 1 if mode == 2 else batch
    name = f"gemm {kind} bn256 {'mn' if mn_major else 'k'} {store} M{M} N{nout} K{K} b{batch}"
    return tk.gemm_case(name, M=M, K=K, nout=nout, batch=batch, bn=256, mn_major=mn_major, mode=mode, act=act, layout=layout,
                        rowscale=rs, store=store, seed=seed, bias=mode != 3)


@pytest.mark.parametrize("store", ["tma", "edge"])
@pytest.mark.parametrize("kind", BN256_KINDS)
def test_gemm_epilogue_tma_choice(monkeypatch, kind, store):
    _run(monkeypatch, kind, store, M=320, K=200, batch=2, seed=11 + BN256_KINDS.index(kind) + 50 * (store == "edge"))


@pytest.mark.parametrize("store", ["tma", "edge"])
def test_gemm_epilogue_tma_mn_major_f32(monkeypatch, store):
    _run(monkeypatch, "store_f32", store, M=320, K=200, batch=3, seed=5, mn_major=True)


@pytest.mark.parametrize("kind", ["resid_f32", "gated_ch_sig_rs", "store_tok"])
def test_gemm_epilogue_tma_many_tiles(monkeypatch, kind):
    """129 x 5 tiles of 64 rows over 132 CTAs: both MMA warpgroups wrap their epilogue chunk rings many times"""
    W = 128 if tk.KINDS[kind][0] == 1 else 256
    _run(monkeypatch, kind, "tma", M=8256, K=136, batch=1, seed=3, nout=5 * W - 8)
