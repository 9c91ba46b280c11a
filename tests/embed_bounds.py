"""fp64 references and per-element error bounds of the template input projections, the pair-init glue and the distogram
head (include/af2b200.h: af2_template_embed[_strict], af2_template_angles[_strict], af2_embed_pair_init, af2_distogram_head).

Plain device-generic torch: test_gpu_embed_heads.py gates the kernels with these bounds on the GPU, and
test_embed_bounds_controls.py checks on the CPU that a faithful emulation of each kernel passes them while plausible wrong
variants do not.  The bounds are derived in test_gpu_embed_heads.py's docstring; u = 2^-24, b = 2^-8.
"""
import torch

from gpu_util import C_GEMM, U32 as U, gemm_f32_bound, gemm_split_bound
from test_gpu_kernels import _act_eps
from test_gpu_strict_kernels import _gelu_ref, _ln_ref

B8 = 2.0 ** -8
GELU_D = 1.13            # max |gelu'(x)| = 1.1289
EPS = 1e-5
GELU = 2                 # _act_eps code of the erf-GELU epilogue


def a8(v):
    return (v + 7) // 8 * 8


def bf(x):
    """fp64 of the round-to-nearest bf16 of fp32 x (what the conversion kernels and the packed weights hold)"""
    return x.bfloat16().double()


def _dot(a, w):
    """a [..., K] @ w [N, K]^T in fp64"""
    return a.double() @ w.double().transpose(0, 1)


# ------------------------------------------------------------------------------------------------------------------------
# A. to_template_embed
# ------------------------------------------------------------------------------------------------------------------------
def template_embed_ref(feats, w, bias, strict):
    """(ref, bound) of t = feats w^T + bias.  bf16: the kernel's operands are bf16(feats) and the packed bf16(w), accumulated
    over align8(K) terms.  strict: three split planes carry the fp32 operands exactly."""
    K = feats.shape[-1]
    a, ww = (feats.double(), w.double()) if strict else (bf(feats), bf(w))
    ref = _dot(a, ww) + bias.double()
    absdot = _dot(a.abs(), ww.abs())
    return ref, (gemm_split_bound if strict else gemm_f32_bound)(absdot, a8(K), ref)


# ------------------------------------------------------------------------------------------------------------------------
# B. template angle MLP: Linear(K, d) -> GELU -> Linear(d, d)
# ------------------------------------------------------------------------------------------------------------------------
def angles_stage1_ref(angles, w1, b1, strict):
    """bf16: h = bf16(gelu(bf16(a) bf16(w1)^T + b1)), the stored GELU epilogue.  strict: h = a w1^T + b1 in fp32 (the GELU is
    applied by the split kernel that feeds stage 2)."""
    K = angles.shape[-1]
    if strict:
        ref = _dot(angles, w1) + b1.double()
        return ref, gemm_split_bound(_dot(angles.abs(), w1.abs()), a8(K), ref)
    ab, wb = bf(angles), bf(w1)
    z = _dot(ab, wb) + b1.double()
    ref = torch.nn.functional.gelu(z)
    e1 = C_GEMM * a8(K) * U * _dot(ab.abs(), wb.abs())
    return ref, B8 * ref.abs() + GELU_D * e1 + _act_eps(z, GELU)


def angles_stage2_ref(h, w2, b2, strict):
    """stage 2 from the kernel's own h.  bf16: h bf16 times bf16(w2).  strict: the exact erf-GELU of the fp32 h, split, times
    the fp32 w2; the GELU kernel's error dg moves each output by at most sum_j |w2_ij| dg_j."""
    d = w2.shape[1]
    if strict:
        g, dg = _gelu_ref(h.double())
        ref = _dot(g, w2) + b2.double()
        return ref, gemm_split_bound(_dot(g.abs() + dg, w2.abs()), d, ref) + _dot(dg, w2.abs())
    hk, wb = h.double(), bf(w2)
    ref = _dot(hk, wb) + b2.double()
    return ref, gemm_f32_bound(_dot(hk.abs(), wb.abs()), d, ref)


def angles_module_ref(angles, w1, b1, w2, b2, strict):
    """(ref, bound) of the whole MLP against the module's fp64 output from its fp32 weights:
        |out - ref| <= sum_j |w2_ij| dh_j + C d u sum_j (|h_j| + dh_j) |w2_ij| + 2 u |ref|      (+ the bf16 weight terms)
    dh is the error of the hidden activation the second GEMM reads.  bf16: dz = (2b + b^2) sum|a w1| (operand roundings)
    + C Kp u (1 + b)^2 sum|a w1| (accumulation), dh = (1 + b) (1.13 dz + eps_gelu(z)) + b |h| (the bf16 store); the packed
    bf16(w2) adds b sum|h w2| and scales the w2 sums by (1 + b).  strict: dz = gemm_split_bound, dh = 1.13 dz + dg(z)."""
    K, d = angles.shape[-1], w2.shape[1]
    z = _dot(angles, w1) + b1.double()
    s1 = _dot(angles.abs(), w1.abs())
    aw2 = w2.double().abs()
    if strict:
        h, dg = _gelu_ref(z)
        dh = GELU_D * gemm_split_bound(s1, a8(K), z) + dg
        ref = _dot(h, w2) + b2.double()
        return ref, _dot(dh, aw2) + gemm_split_bound(_dot(h.abs() + dh, aw2), d, ref)
    h = torch.nn.functional.gelu(z)
    dz = (2 * B8 + B8 * B8) * s1 + C_GEMM * a8(K) * U * (1 + B8) ** 2 * s1
    dh = (1 + B8) * (GELU_D * dz + _act_eps(z, GELU)) + B8 * h.abs()
    ref = _dot(h, w2) + b2.double()
    return ref, ((1 + B8) * _dot(dh, aw2) + B8 * _dot(h.abs(), aw2)
                 + gemm_f32_bound((1 + B8) * _dot(h.abs() + dh, aw2), d, ref))


# ------------------------------------------------------------------------------------------------------------------------
# C. pair init
# ------------------------------------------------------------------------------------------------------------------------
def token_embed(emb, seq, msa, seq_embed=None, msa_embed=None):
    """(e, m) in fp32 with the kernels' operation order: e = emb[seq] (+ seq_embed), m = (emb[msa] (+ msa_embed)) + e.  Every
    add is one IEEE fp32 rounding on either side, so the kernels must match these bitwise."""
    e = emb[seq]
    if seq_embed is not None:
        e = e + seq_embed
    m = emb[msa]
    if msa_embed is not None:
        m = m + msa_embed
    return e, m + e[:, None]


def rel_index(n, R, seq_index=None, device="cpu"):
    idx = torch.arange(n, device=device) if seq_index is None else seq_index.to(device)
    return (idx[:, None] - idx[None, :]).clamp(-R, R) + R


def pair_init_ref(e, w_pair, b_pair, pos, R, seq_index=None, rows=None):
    """(ref, bound) of x[b, i, j] = (l_i + r_j) + pos[clamp(idx_i - idx_j, -R, R) + R] for pair rows i in `rows` (a slice),
    lr = e W^T + b from the fp32 e.  Each lr element is a per-lane fmaf chain of ceil(d/32) terms, 5 shuffle levels and the
    bias add:  dlr <= (ceil(d/32) + 5) u sum|e w| + u |lr|;  x adds two roundings:
        |x - ref| <= (1 + 2u) (dl_i + dr_j) + u |l_i + r_j| + u |ref|."""
    d = e.shape[-1]
    n = e.shape[1]
    rows = slice(0, n) if rows is None else rows
    lr = _dot(e, w_pair) + b_pair.double()
    dlr = ((d + 31) // 32 + 5) * U * _dot(e.abs(), w_pair.abs()) + U * lr.abs()
    l, r, dl, dr = lr[:, rows, None, :d], lr[:, None, :, d:], dlr[:, rows, None, :d], dlr[:, None, :, d:]
    rel = rel_index(n, R, seq_index, e.device)[rows]
    lpr = l + r
    ref = lpr + pos.double()[rel][None]
    return ref, (1 + 2 * U) * (dl + dr) + U * lpr.abs() + U * ref.abs()


# ------------------------------------------------------------------------------------------------------------------------
# D. distogram head
# ------------------------------------------------------------------------------------------------------------------------
def distogram_ref(x, gamma, beta, w, bias, rows=None):
    """(ref, bound) of out[b, i, j] = Linear(LayerNorm((x[b, i, j] + x[b, j, i]) / 2)) for pair rows i in `rows` (a slice).
    One warp per token, VPL = d / 32 values per lane, k_d = VPL + 5 (_ln_ref).  The symmetrised v carries u |v|; through the
    LayerNorm that moves y by |gamma| rstd u (|v| + mean|v| + |xhat| rstd mean(|v - mean| |v|)) (the shift of v and of its
    mean, and the first-order change of the variance).  The Linear is a per-lane fmaf chain + 5 shuffle levels + bias:
        |out - ref| <= sum_k |w_k| dy_k + (VPL + 5) u sum_k (|y_k| + dy_k) |w_k| + u |out|."""
    d = x.shape[-1]
    n = x.shape[1]
    rows = slice(0, n) if rows is None else rows
    v = (x[:, rows].double() + x[:, :, rows].transpose(1, 2).double()) * 0.5
    vpl = d // 32
    g, be = gamma.double(), beta.double()
    y, dy = _ln_ref(v, g, be, vpl + 5, EPS)
    mean = v.mean(-1, keepdim=True)
    xc = v - mean
    rstd = 1.0 / torch.sqrt((xc * xc).mean(-1, keepdim=True) + EPS)
    va = v.abs()
    dy = dy + g.abs() * rstd * U * (va + va.mean(-1, keepdim=True) + (xc * rstd).abs() * rstd * (xc.abs() * va).mean(-1, keepdim=True))
    aw = w.double().abs()
    ref = _dot(y, w) + bias.double()
    return ref, _dot(dy, aw) + (vpl + 5) * U * _dot(y.abs() + dy, aw) + U * ref.abs()


def distogram_inputs(B, n, d, nb, g, device):
    """x with three kinds of pair tokens: unit-scale ones, a block whose symmetrised tokens carry a common offset of ~150 (the
    LayerNorm mean cancels), and a block of tiny spread (variance ~1e-4, where eps = 1e-5 matters)."""
    x = torch.randn(B, n, n, d, generator=g, device=device) * 3
    k = max(1, n // 3)
    x[:, :k] += 300.0
    if n > k:
        x[:, k:, k:] *= 3e-3
    gamma = 1 + 0.5 * torch.randn(d, generator=g, device=device)
    beta = torch.randn(d, generator=g, device=device)
    w = torch.randn(nb, d, generator=g, device=device) * d ** -0.5
    bias = torch.randn(nb, generator=g, device=device)
    return x, gamma, beta, w, bias


def angle_rows_layout(m_before, m_after, row0, T):
    """rows [row0, row0 + T) of every batch element of m [B, m_rows, n, d] all finite, every other row bitwise unchanged"""
    inside = torch.zeros(m_before.shape[1], dtype=torch.bool, device=m_before.device)
    inside[row0:row0 + T] = True
    same = torch.equal(m_before[:, ~inside].view(torch.int32), m_after[:, ~inside].view(torch.int32))
    return same and bool(torch.isfinite(m_after[:, inside]).all())


def within(out, ref, bound):
    """the element-wise gate of gpu_util.check_bound as a predicate (finite and |out - ref| <= bound everywhere)"""
    return bool(torch.isfinite(out).all()) and bool(((out.double() - ref).abs() <= bound).all())
