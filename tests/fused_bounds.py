"""fp64 references and per-element error bounds of the three fused persistent kernels: the GEGLU feed-forward
(csrc/ff_fused.cuh, ff_fused_kernel), the contraction tail (csrc/contract_tail.cuh, contract_tail_kernel) and axial attention
with the q, k, v and gate projections inside the kernel (csrc/attention_proj.cuh, attention_proj_kernel).

Plain device-generic torch: test_gpu_fused_kernels.py gates the kernels with these bounds on the GPU, and
test_fused_bounds_controls.py checks on the CPU that a faithful emulation of each kernel passes them while plausible wrong
variants do not.  Every reference is evaluated in fp64 from the exact bf16 / fp32 operands the kernel is given, and does not
round anywhere; the bound collects the kernel's rounding points.  u = 2^-24 is the fp32 unit roundoff, b = 2^-8 the bf16 one;
E(A, W) = C_GEMM K u |A| |W|^T is the tensor-core accumulation bound of gpu_util.gemm_f32_bound over K terms.

Feed-forward.  x' = x + W2 h + b2,  h = (u + b_u) gelu(g + b_g),  [u | g] = W1 xn over D (W1 and b1 as pack_feed_forward
packs them: per 128 hidden units 128 value rows, then 128 gate rows).  GEMM 1 and the GEGLU are the gated epilogue of
test_gpu_kernels.py, with the + b and the product roundings added:
    E_u = E(xn, W_u) + u |u + b_u|,   E_g = E(xn, W_g) + u |g + b_g|
    dh  = |gelu(g + b_g)| E_u + |u + b_u| (1.13 E_g + eps_gelu(g + b_g)) + u |h|          (eps_gelu: test_gpu_kernels._act_eps)
    dh += b (|h| + dh)                                                                    (bf16 store of h)
GEMM 2 accumulates the stored h over `hidden` terms, then adds b2 and x (two fp32 roundings):
    e   = dh |W2|^T + C_GEMM hidden u (|h| + dh) |W2|^T + 2 u (|y| + e_h)                 (y = W2 h + b2, e_h = dh |W2|^T)
    |x' - ref| <= e + u (|ref| + e)

Contraction tail.  x' = x + W_out t + b_out over D, with t as chan_to_token makes it:
  CT_SCALE: t = bf16(O s), s the fp32 per-token scale or fl(scale_const): dt = (b + 2 u) |O s| (test_gpu_contractions._c2t_ref).
  gated:    t = bf16(LN(O) gate), LN(O) = (O - mean) rstd gamma + beta over the D channels.  The LayerNorm bound e_LN is
            _c2t_ref's with gate 1 (two-pass fp32 moments over a tree of depth k_d, rsqrtf, three fp32 roundings), whose
            store term b |LN| is taken off again.  CT_GATE_LOAD reads the bf16 gate exactly; CT_GATE_PROJECT computes it as
                gate = bf16(sigmoid(xn W_og^T + b_og)):  dg = 1/4 (E(xn, W_og) + u |z|) + 1e-6 sigmoid(z),  dg += b (gate + dg)
            (z = xn W_og^T + b_og, 1/4 = max sigmoid', 1e-6 sigmoidf_fast's relative error), so
                dt = (|gate| + dg) e_LN + |LN| dg,  dt += b (|t| + dt)
  then GEMM 2 over D terms and the + b_out, + x roundings as the feed-forward:
    e = dt |W_out|^T + C_GEMM D u (|t| + dt) |W_out|^T + 2 u (|y| + e_t),  |x' - ref| <= e + u (|ref| + e)

Projected attention.  q | k | v = xn W_qkv^T (the q rows carry dim_head^-0.5 log2 e, so the logits are in the log2 domain),
gate = sigmoid(xn W_g^T + b_g), and the module's attention: s = q k^T + bias, s.masked_fill(~(mask_q & mask_k), -max),
p = softmax_2(s) over the n keys (a fully masked query row averages all n values: quirk Q1), out = (p v) gate.  The kernel
rounds q, k, v and the gate to bf16 as the projection GEMM's epilogues do:
    dq, dk, dv = E(xn, W) + b (|.| + E(xn, W)),     dg as the tail's projected gate
    ds_ij = sum_e (|dq| |k| + |q| |dk| + |dq| |dk|)_e + dh u sum_e (|q| + |dq|)_e (|k| + |dk|)_e + u (|s_ij| + ds_ij)
(the rounded operands, plus the fp32 logit accumulation and the + bias rounding).  With delta_i = max over the valid keys j of
ds_ij, every weight p_j = 2^{s_j} / sum 2^{s_l} moves by a factor within 2^{+-2 delta_i}, so
    |do| <= (2^{2 delta} - 1) sum_j p_j |v_j| + 2^{2 delta} sum_j p_j |dv_j|,     E = |do| (|g| + dg) + |o| dg
and on top of that the attention kernel's own rounding (test_gpu_attention_kernel.attention_ref: the bf16 store of the
output and the bf16 rounding of P against the fp32 normaliser), evaluated with the perturbed magnitudes:
    |out - ref| <= E + b (|ref| + E) + C_ATTN b (|g| + dg) 2^{2 delta} sum_j p_j (|v_j| + |dv_j|)
Fully masked query rows take no logit at all (delta = 0) and average the rounded v.  The fp64 temporaries are bounded by
working on chunks of folded rows, as attention_ref does.
"""
import math

import torch

from gpu_util import C_GEMM, U32 as U, gemm_f32_bound
from test_gpu_attention_kernel import C_ATTN, NEG
from test_gpu_contractions import _c2t_ref
from test_gpu_kernels import _act_eps

B8 = 2.0 ** -8
GELU_D = 1.13            # max |gelu'(x)| = 1.1289
SIG_D = 0.25             # max sigmoid'(x)
EPS = 1e-5
GELU, SIGMOID = 2, 1     # _act_eps codes


def _mm(a, w):
    """a [..., K] @ w [N, K]^T in fp64"""
    return a.double() @ w.double().transpose(0, 1)


def _proj(a, w, bias=None):
    """fp64 projection of the bf16 operands and its accumulation bound: (a w^T [+ bias], E(a, w) [+ u |a w^T + bias|])"""
    K = a.shape[-1]
    p = _mm(a, w)
    e = C_GEMM * K * U * _mm(a.abs(), w.abs())
    if bias is not None:
        p = p + bias.double()
        e = e + U * p.abs()
    return p, e


def _resid_out(t, dt, w_out, b_out, x):
    """(x + t w_out^T + b_out, bound) for the fp32-accumulated GEMM over t (exact t with error dt, as the kernel holds it)"""
    K = t.shape[-1]
    wa = w_out.double().abs()
    y = _mm(t, w_out) + (0.0 if b_out is None else b_out.double())
    e_t = dt @ wa.transpose(0, 1)
    e = e_t + gemm_f32_bound((t.abs() + dt) @ wa.transpose(0, 1), K, y.abs() + e_t)
    ref = x.double() + y
    return ref, e + U * (ref.abs() + e)


# ------------------------------------------------------------------------------------------------------------------------
# feed-forward
# ------------------------------------------------------------------------------------------------------------------------
def unpack_w1(w1, b1):
    """the packed W1 [2 hidden, D] / b1 [2 hidden] (per 128 hidden units: 128 value rows, 128 gate rows) -> value and gate
    halves in hidden order"""
    D = w1.shape[-1]
    tiles = w1.shape[0] // 256
    w = w1.view(tiles, 2, 128, D)
    b = b1.view(tiles, 2, 128)
    return w[:, 0].reshape(-1, D), w[:, 1].reshape(-1, D), b[:, 0].reshape(-1), b[:, 1].reshape(-1)


def ff_ref(x, xn, w1, b1, w2, b2, rows=8192):
    """(x + W2 h + b2, bound) fp64 [T, D] for x fp32 [T, D], xn bf16 [T, D] and the packed w1 / b1, w2 bf16 [D, hidden], b2"""
    T, D = xn.shape
    wu, wg, bu, bg = unpack_w1(w1, b1)
    out = torch.empty(T, D, dtype=torch.float64, device=xn.device)
    bnd = torch.empty_like(out)
    for r0 in range(0, T, rows):
        a = xn[r0:r0 + rows]
        uu, eu = _proj(a, wu, bu)
        gg, eg = _proj(a, wg, bg)
        act = torch.nn.functional.gelu(gg)
        h = uu * act
        dh = act.abs() * eu + uu.abs() * (GELU_D * eg + _act_eps(gg, GELU)) + U * h.abs()
        dh = dh + B8 * (h.abs() + dh)
        o, e = _resid_out(h, dh, w2, b2, x[r0:r0 + rows])
        out[r0:r0 + rows] = o
        bnd[r0:r0 + rows] = e
    return out, bnd


# ------------------------------------------------------------------------------------------------------------------------
# contraction tail
# ------------------------------------------------------------------------------------------------------------------------
def tail_gate_ref(xn, w_og, b_og):
    """(sigmoid(xn w_og^T + b_og), bound of the kernel's bf16 gate) fp64 [T, D]"""
    z, ez = _proj(xn, w_og, b_og)
    g = torch.sigmoid(z)
    dg = SIG_D * ez + _act_eps(z, SIGMOID)
    return g, dg + B8 * (g + dg)


def tail_ref(O, x, w_out, b_out, *, gamma=None, beta=None, gate=None, xn=None, w_og=None, b_og=None, scale=None,
             scale_const=None, rows=16384):
    """(x + tail(O) w_out^T + b_out, bound) fp64 [T, D].  O fp32 [T, D] (token-major view of the contraction output), x fp32.
    Gated (gamma, beta given): the bf16 gate [T, D] as loaded, or xn / w_og / b_og to project it.  Otherwise the scale:
    the fp32 per-token scale [T] or scale_const."""
    T, D = O.shape
    out = torch.empty(T, D, dtype=torch.float64, device=O.device)
    bnd = torch.empty_like(out)
    for r0 in range(0, T, rows):
        sl = slice(r0, r0 + rows)
        o = O[sl]
        if gamma is None:
            s = (scale[sl] if scale is not None else
                 torch.full((o.shape[0],), scale_const, dtype=torch.float32, device=o.device))
            t, dt = _c2t_ref(D, "scale", dict(x=o.t(), scale=s))
        else:
            if xn is not None:
                g, dg = tail_gate_ref(xn[sl], w_og, b_og)
            else:
                g, dg = gate[sl].double(), torch.zeros((), dtype=torch.float64, device=o.device)
            one = torch.ones(o.shape, dtype=torch.float64, device=o.device)
            ln, e1 = _c2t_ref(D, "ln", dict(x=o.t(), gamma=gamma, beta=beta, gate=one))
            e_ln = e1 - B8 * ln.abs()
            t = ln * g
            dt = (g.abs() + dg) * e_ln + ln.abs() * dg
            dt = dt + B8 * (t.abs() + dt)
        r, e = _resid_out(t, dt, w_out, b_out, x[sl])
        out[sl] = r
        bnd[sl] = e
    return out, bnd


# ------------------------------------------------------------------------------------------------------------------------
# projected attention
# ------------------------------------------------------------------------------------------------------------------------
def attention_proj_ref(xn, wqkv, wg, bg, bias, mask_bn, n, nbatch, heads, dh, idx, elems=1 << 24):
    """fp64 reference (module semantics) of af2_attention_proj_bf16 and its bound, both [tokens, heads * dh] on xn's device.
    idx [nbatch, n]: token of (folded row b, position i); mask_bn [nbatch, n] bool or None; bias bf16 [heads, n, align8(n)]
    (log2 domain) or None"""
    I = heads * dh
    T, d = xn.shape
    dev = xn.device
    out = torch.empty(T, I, dtype=torch.float64, device=dev)
    bnd = torch.empty_like(out)
    wq, wk, wv = wqkv[:I], wqkv[I:2 * I], wqkv[2 * I:]
    chunk = max(1, elems // (heads * n * n))
    for b0 in range(0, nbatch, chunk):
        ix = idx[b0:b0 + chunk].to(dev)
        nb = ix.shape[0]
        a = xn[ix.flatten()]
        hv = lambda t: t.view(nb, n, heads, dh).permute(0, 2, 1, 3)   # noqa: E731  [nb, H, n, dh]
        parts = []
        for w in (wq, wk, wv):
            p, e = _proj(a, w)
            parts += [hv(p), hv(e + B8 * (p.abs() + e))]
        q, dq, k, dk, v, dv = parts
        g, dg = tail_gate_ref(a, wg, bg)
        g, dg = hv(g), hv(dg)
        s = q @ k.transpose(-1, -2)
        qk = q.abs() @ k.abs().transpose(-1, -2)
        ps = (q.abs() + dq) @ (k.abs() + dk).transpose(-1, -2)
        ds = (ps - qk) + dh * U * ps
        if bias is not None:
            s = s + bias[:, :, :n].double().to(dev)[None]
        ds = ds + U * (s.abs() + ds)
        if mask_bn is not None:
            m = mask_bn[b0:b0 + nb].to(dev)
            pair = m[:, None, :, None] & m[:, None, None, :]
            s = s.masked_fill(~pair, NEG)
            ds = ds.masked_fill(~pair, 0.0)
        delta = ds.amax(-1, keepdim=True)
        f = torch.exp2(2 * delta)
        p = torch.softmax(s * math.log(2.0), dim=-1)
        o = p @ v
        pv = p @ v.abs()
        pdv = p @ dv
        do = (f - 1) * pv + f * pdv
        r = o * g
        e = do * (g.abs() + dg) + o.abs() * dg
        e = e + B8 * (r.abs() + e) + C_ATTN * B8 * (g.abs() + dg) * f * (pv + pdv)
        tok = ix.flatten()
        out[tok] = r.permute(0, 2, 1, 3).reshape(-1, I)
        bnd[tok] = e.permute(0, 2, 1, 3).reshape(-1, I)
    return out, bnd


def within(out, ref, bound):
    """every element finite and within its bound (the CPU controls' form of gpu_util.check_bound)"""
    out = out.double()
    return bool(torch.isfinite(out).all()) and bool(((out - ref).abs() <= bound).all())
