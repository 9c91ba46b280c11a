"""Device time of Attention.forward called on its own (alphafold2_b200.Attention, alphafold2.py:125-190) against the
reference's eager lines on the same card:
   python tools/time_attention_forward.py [--calls 20] [--rounds 3]
   -> one JSON line per shape and round, then one summary line

Shapes (bf16 mode, heads 8, dim_head 64, d 256, masks given, 20 % of the keys masked):
  self      B 256, i = j 256, a [1, h, i, j] bias    (an axial-attention fold)
  cross     B 256, i 256, j 64, a context mask       (cross-attention)
  template  B 65,536, i 1, j 4, a context mask       (the pointwise template call of alphafold2.py:767-772)
Each call is timed with CUDA events (L2 flushed before it); `eager` is the reference's Attention.forward lines in PyTorch
bf16 (Linear layers, einsum, masked_fill, softmax, einsum, gate, to_out) on the same inputs and weights.  For the self
shape the attention core alone (attention_tc_kernel<64, true>, the library's per-launch events of the attention class
inside Attention.forward) is also timed against ops.attention_bf16 (attention_tc_kernel<64>) on a q|k|v and gate of the
same shapes with the same bias and mask.  The rounds alternate the implementations so that the run-to-run spread is
visible.  The card name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import alphafold2_b200 as A  # noqa: E402
from alphafold2_b200 import _lib, ops  # noqa: E402

KC_ATTENTION = 2
SHAPES = {"self": (256, 256, 256, True), "cross": (256, 256, 64, False), "template": (65536, 1, 4, False)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl = [v.strip() for v in q.split(",")]
        return dict(name=name, power_limit=pl)
    except Exception as e:  # noqa: BLE001
        return dict(name=torch.cuda.get_device_name(), error=str(e))


def eager(mod, x, mask, bias, context, context_mask):
    """alphafold2.py:125-190 in bf16 (the reference's own lines, dropout off)"""
    h = mod.heads
    c = x if context is None else context
    q, k, v = mod.to_q(x), *mod.to_kv(c).chunk(2, dim=-1)
    q, k, v = (t.reshape(t.shape[0], t.shape[1], h, -1).permute(0, 2, 1, 3) for t in (q, k, v))
    dots = torch.einsum("bhid,bhjd->bhij", q * mod.scale, k)
    if bias is not None:
        dots = dots + bias
    cm = mask if context is None else context_mask
    dots = dots.masked_fill(~(mask[:, None, :, None] & cm[:, None, None, :]), -torch.finfo(dots.dtype).max)
    out = torch.einsum("bhij,bhjd->bhid", dots.softmax(dim=-1), v).permute(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], -1)
    return mod.to_out(out * mod.gating(x).sigmoid())


def events(fn, flush, calls):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(calls):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        total += e0.elapsed_time(e1)
    return total / calls


def profiled(lib, fn, flush, calls):
    """mean device time of the attention-class launches inside fn (the library's per-launch CUDA events)"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    lib.af2_profile_enable(1)
    for _ in range(calls):
        flush.zero_()
        fn()
    ms = C.c_double()
    cnt = lib.af2_profile_read(KC_ATTENTION, C.byref(ms), None, None)
    lib.af2_profile_enable(0)
    if cnt != calls:
        raise RuntimeError(f"expected {calls} attention launches, the profile recorded {cnt}")
    return ms.value / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = _lib.load()
    d, heads, dh = 256, 8, 64
    I = heads * dh
    flush = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    mod = A.Attention(d, heads=heads, dim_head=dh).cuda().eval()
    torch.nn.init.normal_(mod.to_out.weight, std=0.02)
    ref = A.Attention(d, heads=heads, dim_head=dh).cuda().eval()
    ref.load_state_dict(mod.state_dict())
    ref = ref.to(torch.bfloat16)
    summary = dict(card=card())
    with torch.no_grad():
        for name, (B, i, j, self_attn) in SHAPES.items():
            g = torch.Generator(device="cuda").manual_seed(B + i + j)
            x = torch.randn(B, i, d, device="cuda", generator=g)
            context = None if self_attn else torch.randn(B, j, d, device="cuda", generator=g)
            mask = torch.rand(B, i, device="cuda", generator=g) > 0.2
            cmask = None if self_attn else torch.rand(B, j, device="cuda", generator=g) > 0.2
            bias = torch.randn(1, heads, i, j, device="cuda", generator=g) if self_attn else None
            xb, cb, bb = x.bfloat16(), None if context is None else context.bfloat16(), None if bias is None else bias.bfloat16()
            ours_fn = lambda: mod(x, mask=mask, attn_bias=bias, context=context, context_mask=cmask)  # noqa: E731
            ref_fn = lambda: eager(ref, xb, mask, bb, cb, cmask)  # noqa: E731
            out = ours_fn().double()
            diff = (out - ref_fn().double()).abs().max().item() / out.pow(2).mean().sqrt().item()
            rows = []
            for r in range(args.rounds):
                row = dict(shape=name, round=r, B=B, i=i, j=j, ms=events(ours_fn, flush, args.calls),
                           eager_ms=events(ref_fn, flush, args.calls))
                if self_attn:
                    qkv = torch.randn(B * i, 3 * I, device="cuda", generator=g).bfloat16()
                    gate = torch.rand(B * i, I, device="cuda", generator=g).bfloat16()
                    bt = torch.zeros(heads, i, (j + 7) // 8 * 8, device="cuda", dtype=torch.bfloat16)
                    bt[:, :, :j] = (bias[0] * 1.4426950408889634).bfloat16()
                    m = mask.reshape(-1)
                    row["core_ms"] = profiled(lib, ours_fn, flush, args.calls)
                    row["attention_bf16_ms"] = profiled(
                        lib, lambda: ops.attention_bf16(qkv, gate, i, B, heads, dh, i, 1, bias=bt, mask=m), flush, args.calls)
                row["speedup_vs_eager"] = row["eager_ms"] / row["ms"]
                rows.append(row)
                print(json.dumps(row), flush=True)
            summary[name] = dict(ms=min(r["ms"] for r in rows), eager_ms=min(r["eager_ms"] for r in rows),
                                 max_rel_diff_vs_eager_bf16=diff)
            if self_attn:
                summary[name]["core_ms"] = [r["core_ms"] for r in rows]
                summary[name]["attention_bf16_ms"] = [r["attention_bf16_ms"] for r in rows]
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
