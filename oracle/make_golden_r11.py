"""TEST INFRASTRUCTURE ONLY -- round-11 fixture from the UNMODIFIED reference (run in the dev container):
    python -m oracle.make_golden_r11
  tests/golden/distogram_loss.pt  alphafold2_pytorch/utils.py's get_bucketed_distance_matrix and the loss lines of
  train_pre.py:76-90 (F.cross_entropy of the permuted distogram, ignore_index), run on the CPU in fp32, per case:
    small     b 2, N 20, nb 37 (torch.cdist is direct up to 25 points): masked residues, a NaN coordinate of an unmasked
              residue, and residues on a line whose distances fall exactly on the edges 2.0, 2.5, ..., 8.0
    edges16   b 2, N 18, nb 16: residues on a line at the fp32 edges themselves (torch.linspace(2, 20, 16) is not exact in
              binary), so the distances from residue 0 are exactly those edges
    masked    b 3, N 12, nb 37: element 1 fully masked (the batch mean runs over elements 0 and 2)
    large     b 1, N 27, nb 37 (cdist's |a|^2 + |b|^2 - 2 a.b form): every distance at least 0.05 A from an edge
    large16   b 2, N 28, nb 16: the same at another bucket count
  and the small case again with ignore_index 3 (a bucket index: the pairs in bucket 3 drop out too).
  Random distances everywhere are resampled until they lie at least MARGIN from every edge, so a one-ulp difference between
  the reference's distance and the direct fp32 one cannot change a label.  Under 500 KB."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_loader import load_reference  # noqa: E402
from oracle.make_golden import OUT  # noqa: E402

MARGIN = 0.05


def far(d, edges):
    d = d[torch.isfinite(d)]
    return bool(((d[:, None] - edges[None]).abs() >= MARGIN).all())


def coords_far(b, n, nb, g, scale):
    """[b, n, 3] random points added one at a time, each resampled until its distances to the earlier ones are MARGIN from
    every edge"""
    edges = torch.linspace(2, 20, steps=nb).double()
    x = torch.empty(b, n, 3)
    for e in range(b):
        for i in range(n):
            while True:
                p = torch.randn(3, generator=g) * scale
                if far((x[e, :i].double() - p.double()).pow(2).sum(-1).sqrt(), edges):
                    x[e, i] = p
                    break
    return x


def main():
    load_reference()
    import torch.nn.functional as F
    from einops import rearrange
    import alphafold2_pytorch.utils as U

    g = torch.Generator().manual_seed(11)

    def run(coords, mask, logits, nb, ignore_index=-100):
        labels = U.get_bucketed_distance_matrix(coords, mask, nb, ignore_index)
        loss = F.cross_entropy(rearrange(logits, 'b i j c -> b c i j'), labels, ignore_index=ignore_index)
        return {"coords": coords, "mask": mask, "logits": logits, "nb": nb, "ignore_index": ignore_index, "labels": labels,
                "loss": loss}

    fx = {}
    # small: random residues, then 13 on a line (element 0: 0.5 A apart, element 1: 1 A apart), distances on the edges
    n, nb = 20, 37
    x = coords_far(2, n, nb, g, 4.0)
    line = torch.arange(13, dtype=torch.float32) * 0.5                 # 0, 0.5, ..., 6.0: differences are multiples of 0.5
    x[0, 7:, :] = 0.0
    x[0, 7:, 0] = line + 30.0
    x[1, 7:, :] = 0.0
    x[1, 7:, 1] = line * 2 - 40.0                                      # 0, 1, ..., 12: every difference an edge or between
    x[1, 3, 2] = float("nan")                                          # unmasked: label nb - 1 against everything
    mask = torch.ones(2, n, dtype=torch.bool)
    mask[0, 2] = mask[0, 5] = mask[1, 0] = False
    logits = torch.randn(2, n, n, nb, generator=g) * 3
    fx["small"] = run(x, mask, logits, nb)
    fx["small_ignore3"] = run(x, mask, logits, nb, ignore_index=3)
    # edges16: distances from residue 0 exactly the fp32 edges of linspace(2, 20, 16)
    n, nb = 18, 16
    x = coords_far(2, n, nb, g, 4.0)
    edges = torch.linspace(2, 20, steps=nb)
    x[:, :16, :] = 0.0
    x[:, 1:16, 0] = edges[:15]
    x[1, :16, :] = x[1, :16, :].roll(1, dims=-1)                       # along y in element 1
    mask = torch.ones(2, n, dtype=torch.bool)
    mask[1, 17] = False
    fx["edges16"] = run(x, mask, torch.randn(2, n, n, nb, generator=g) * 2, nb)
    # masked: element 1 has no residue
    n, nb = 12, 37
    x = coords_far(3, n, nb, g, 5.0)
    mask = torch.rand(3, n, generator=g) > 0.25
    mask[1] = False
    mask[0, 0] = mask[2, 0] = True
    fx["masked"] = run(x, mask, torch.randn(3, n, n, nb, generator=g) * 3, nb)
    # large: the matrix form of cdist, distances away from the edges; coordinates well away from the origin
    n, nb = 27, 37
    x = coords_far(1, n, nb, g, 6.0) + 25.0
    mask = torch.ones(1, n, dtype=torch.bool)
    mask[0, -3:] = False
    fx["large"] = run(x, mask, torch.randn(1, n, n, nb, generator=g) * 3, nb)
    n, nb = 28, 16
    x = coords_far(2, n, nb, g, 8.0)
    mask = torch.rand(2, n, generator=g) > 0.2
    fx["large16"] = run(x, mask, torch.randn(2, n, n, nb, generator=g) * 3, nb)
    path = os.path.join(OUT, "distogram_loss.pt")
    torch.save(fx, path)
    print(f"wrote distogram_loss ({os.path.getsize(path)} bytes)")
    for k, v in fx.items():
        print(f"  {k}: loss {v['loss'].item():.6f}, counted {(v['labels'] != v['ignore_index']).sum().item()}")


if __name__ == "__main__":
    main()
