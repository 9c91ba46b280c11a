"""-m gpu: tied-query column attention split over column shards, af2_axial_attention_tied_begin / _end (include/af2b200.h).

The sharded schedule holds a column shard of the pair tensor per rank, while the tied queries of the extra-MSA stack average
over all columns.  Here one process plays every shard: each piece of columns runs _begin into its own workspace, the
pieces' fp32 query sums are concatenated in column order (what the schedule's all-gather delivers), and each piece runs
_end.  Gates:
  * one piece holding every column: bitwise equal to af2_axial_attention_ex(flags = 1) with the same bias;
  * 2, 3 and 4 uneven pieces: within 2e-3 * max|x| of that whole call, and check() of the attention's update against the
    fp64 oracle (O.attention with tie_dim = all columns);
  * every malformed call returns AF2_ERR_BAD_ARG."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# d, heads, dim_head, h (attended rows; 37 and 61 are not multiples of 8), w (columns), masked
CASES = [
    (64, 2, 32, 37, 12, True),
    (128, 4, 32, 48, 9, False),
    (128, 2, 64, 61, 7, True),
    (256, 4, 64, 40, 10, False),
]
SPLITS = [[0, 5, None], [0, 2, 6, None], [0, 1, 3, 4, None]]     # column offsets of 2, 3 and 4 uneven pieces (None: w)


def _setup(d, H, dh, h, w, masked):
    import alphafold2_b200 as A
    from oracle import evoformer_oracle as O
    torch.manual_seed(d + h + w)
    ax = A.AxialAttention(dim=d, heads=H, dim_head=dh, row_attn=False, col_attn=True, accept_edges=True, global_query_attn=True)
    st = O.randomize_zero_init_({k: v.clone() for k, v in ax.state_dict().items()}, std=0.05)
    ax.load_state_dict(st)
    ax = ax.cuda().eval()
    x = torch.randn(h, w, d, device="cuda")
    edges = torch.randn(h, h, d, device="cuda")
    mask = None
    if masked:
        mask = torch.rand(h, w, device="cuda") > 0.15
        mask[:, 0] = True
    return ax, st, x, edges, mask


def _whole(ax, x, edges, mask):
    """af2_axial_attention_ex(flags = 1) on a copy of x [h, w, d]."""
    from alphafold2_b200 import _lib, ops
    h, w, d = x.shape
    out = x.clone()
    lib = _lib.load()
    ws = ops.workspace(lib.af2_axial_attention_workspace(1, h, w, d, ax.attn.heads, ax.attn.dim_head, 0), x.device)
    _lib.check(lib.af2_axial_attention_ex(C.byref(ax.packed().struct), out.data_ptr(), edges.data_ptr(),
                                          None if mask is None else mask.contiguous().data_ptr(), 1, h, w, d, ax.attn.heads,
                                          ax.attn.dim_head, 0, 1, ws.data_ptr(), ws.numel(), ops._stream_ptr()))
    return out


def _pieces(ax, x, bias, mask, offs):
    """begin for every column piece (own workspace), the sums concatenated in column order, end for every piece."""
    from alphafold2_b200 import _lib, ops
    lib = _lib.load()
    h, w, d = x.shape
    H, dh = ax.attn.heads, ax.attn.dim_head
    s = ops._stream_ptr()
    runs = []
    for c0, c1 in zip(offs, offs[1:]):
        xp = x[:, c0:c1].contiguous().clone()                      # never x itself: x stays the input of every split
        mp_ = None if mask is None else mask[:, c0:c1].contiguous()
        ws = torch.empty(lib.af2_axial_attention_workspace(1, h, c1 - c0, d, H, dh, 0), dtype=torch.uint8, device=x.device)
        qsum = torch.empty(h, H * dh, dtype=torch.float32, device=x.device)
        args = (C.byref(ax.packed().struct), xp.data_ptr(), bias.data_ptr(), None if mp_ is None else mp_.data_ptr(), h, c1 - c0,
                d, H, dh)
        _lib.check(lib.af2_axial_attention_tied_begin(*args, qsum.data_ptr(), ws.data_ptr(), ws.numel(), s))
        runs.append((xp, args, ws, qsum, mp_))
    parts = torch.cat([r[3] for r in runs]).contiguous()
    for xp, args, ws, _, _ in runs:
        _lib.check(lib.af2_axial_attention_tied_end(*args, parts.data_ptr(), len(runs), w, ws.data_ptr(), ws.numel(), s))
    return torch.cat([r[0] for r in runs], 1)


def _oracle_update(st, x, edges, mask, H):
    """fp64: the tied column attention's update of x [h, w, d] (alphafold2.py:142-151, 192-255)."""
    from gpu_util import to64
    from oracle import evoformer_oracle as O
    w = to64(st)
    x64, e64 = x.double().cpu(), edges.double().cpu()
    xn = F.layer_norm(x64, (x64.shape[-1],), w["norm.weight"], w["norm.bias"], 1e-5).transpose(0, 1).contiguous()   # [w, h, d]
    bias = torch.einsum("ijd,hd->hij", e64, w["edges_to_attn_bias.0.weight"])[None]
    mk = None if mask is None else mask.cpu().transpose(0, 1).contiguous()
    return O.attention(w, "attn.", xn, H, mk, bias, tie_dim=x.shape[1]).transpose(0, 1)


@pytest.mark.parametrize("d,H,dh,h,w,masked", CASES)
def test_tied_parts(d, H, dh, h, w, masked):
    from alphafold2_b200.stages import CudaStageOps
    from gpu_util import check
    ax, st, x, edges, mask = _setup(d, H, dh, h, w, masked)
    whole = _whole(ax, x, edges, mask)
    bias = CudaStageOps().pair_bias(ax, edges)                      # [H, h, align8(h)], the kernel the whole call runs
    one = _pieces(ax, x, bias, mask, [0, w])
    torch.cuda.synchronize()
    assert torch.equal(one, whole), f"one piece differs from af2_axial_attention_ex(flags=1): {(one - whole).abs().max().item():.3e}"
    ref = _oracle_update(st, x, edges, mask, H)
    scale = whole.abs().max().item()
    for offs in SPLITS:
        offs = offs[:-1] + [w]
        out = _pieces(ax, x, bias, mask, offs)
        err = (out - whole).abs().max().item()
        print(f"tied parts d={d} h={h} w={w} pieces={len(offs) - 1}: {err / scale:.3e} max|x| from the whole call")
        assert err <= 2e-3 * scale, (offs, err, scale)
        check(f"tied_parts/d{d}h{h}w{w}/{len(offs) - 1}", (out - x).cpu(), ref)


def test_tied_parts_reject_bad_arguments():
    from alphafold2_b200 import _lib, ops
    lib = _lib.load()
    d, H, dh, h, w = 64, 2, 32, 16, 4
    ax, _, x, edges, _ = _setup(d, H, dh, h, w, False)
    pk = C.byref(ax.packed().struct)
    ws = torch.empty(lib.af2_axial_attention_workspace(1, h, w, d, H, dh, 0), dtype=torch.uint8, device="cuda")
    qs = torch.zeros(h, H * dh, device="cuda")
    s = ops._stream_ptr()
    x0 = x.clone()

    def begin(pk=pk, x=x.data_ptr(), hh=h, ww=w, q=qs.data_ptr(), wsp=ws.data_ptr()):
        return lib.af2_axial_attention_tied_begin(pk, x, None, None, hh, ww, d, H, dh, q, wsp, ws.numel(), s)

    def end(pk=pk, x=x.data_ptr(), hh=h, ww=w, parts=qs.data_ptr(), nparts=1, ncols=w, wsp=ws.data_ptr()):
        return lib.af2_axial_attention_tied_end(pk, x, None, None, hh, ww, d, H, dh, parts, nparts, ncols, wsp, ws.numel(), s)

    bad = [begin(pk=None), begin(x=None), begin(q=None), begin(wsp=None), begin(hh=0), begin(ww=0),
           end(pk=None), end(x=None), end(parts=None), end(wsp=None), end(hh=0), end(ww=0), end(nparts=0), end(nparts=-2),
           end(ncols=w - 1)]
    torch.cuda.synchronize()
    assert bad == [-1] * len(bad), bad
    assert torch.equal(x, x0), "a rejected call wrote x"
