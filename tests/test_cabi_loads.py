"""CPU: the C-ABI library builds/loads and exports every symbol include/af2b200.h declares (no compute calls)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from alphafold2_b200 import _lib
    if not os.path.isfile(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "af2b200.h")).read()
    names = set(re.findall(r"\b(af2_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 14
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/af2b200.h but not exported"
    from alphafold2_b200 import _lib
    assert names == set(_lib.EXPORTED_SYMBOLS)


def test_abi_version(lib):
    assert lib.af2_abi_version() == 3
    assert lib.af2_last_error() is not None


def test_workspace_queries(lib):
    assert lib.af2_feed_forward_workspace(1024, 256, 1024) > 1024 * 256 * 2
    assert lib.af2_axial_attention_workspace(1, 128, 256, 256, 8, 64, 1) > 0
    assert lib.af2_triangle_multiply_workspace(1, 256, 256) > 0
    assert lib.af2_outer_mean_workspace(1, 128, 256, 256) > 0


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "alphafold2_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f"{f} imports the oracle"


def test_state_dict_keys_match_reference_fixture():
    """tests/golden/alphafold2_state_keys.json is the FULL state_dict of the unmodified reference (oracle/make_golden_keys.py)
    for two constructor configurations: the drop-in must have exactly the same keys and shapes, and the same zero / one
    initialisation (quirk Q8), key by key.  (`ipa_block.*` of a real checkpoint is third-party, not mirrored: load such a
    checkpoint with strict=False.)"""
    import json
    import torch
    import alphafold2_b200 as A
    from conftest import GOLDEN
    spec = json.load(open(os.path.join(GOLDEN, "alphafold2_state_keys.json")))
    for name, entry in spec.items():
        torch.manual_seed(0)
        model = A.Alphafold2(**entry["cfg"])
        ours = model.state_dict()
        ref = entry["keys"]
        assert set(ours) == set(ref), (name, sorted(set(ours) ^ set(ref))[:10])
        for k, info in ref.items():
            v = ours[k]
            assert list(v.shape) == info["shape"], (name, k, list(v.shape), info["shape"])
            if info["init"] == "zeros":
                assert bool((v == 0).all()), (name, k, "reference initialises this tensor to zero")
            elif info["init"] == "ones":
                assert bool((v == 1).all()), (name, k, "reference initialises this tensor to one")
            elif torch.is_floating_point(v) and v.numel() > 1:
                assert not bool((v == 0).all()) and not bool((v == 1).all()), (name, k, "reference uses a random init here")
    from conftest import load_golden
    fx = load_golden("evoformer_block")
    c = fx["cfg"]
    blk = A.EvoformerBlock(dim=c["dim"], seq_len=c["N"], heads=c["heads"], dim_head=c["dim_head"], attn_dropout=0., ff_dropout=0.)
    blk.load_state_dict(fx["state"], strict=True)


def test_packed_cache_invalidation_and_copy():
    """ADVICE r1: the packed-weight cache must follow parameter updates it can see (copy_, load_state_dict, eval()/train(),
    .to()), expose invalidate_packed() for writes through .data, and never travel with deepcopy / pickle."""
    import copy
    import io
    import torch
    import alphafold2_b200 as A
    from alphafold2_b200.alphafold2 import _Packable

    class Probe(_Packable):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(4, 4)
            self.count = 0

        def _pack(self):
            self.count += 1
            return ("packed", float(self.lin.weight.detach().sum()))

    p = Probe()
    a = p.packed()
    assert p.packed() is a and p.count == 1
    with torch.no_grad():
        p.lin.weight.add_(1.0)                              # version bump -> repack
    assert p.packed() is not a and p.count == 2
    p.load_state_dict({k: v.clone() for k, v in p.state_dict().items()})
    p.packed()
    assert p.count == 3
    p.eval()
    p.packed()
    assert p.count == 4
    p.lin.weight.data.mul_(2.0)                             # invisible to (data_ptr, _version) ...
    stale = p.packed()
    assert p.count == 4 and stale[1] != float(p.lin.weight.detach().sum())
    A.invalidate_packed(p)                                  # ... so the documented hook is needed
    assert p.packed()[1] == float(p.lin.weight.detach().sum()) and p.count == 5
    q = copy.deepcopy(p)
    assert "_pk" not in q.__dict__ and q.count == 5
    A.set_precision(p, "strict")                            # precision is part of the key
    p.packed()
    assert p.count == 6
    ff = A.FeedForward(dim=32)
    ff.__dict__["_pk"] = lambda: None                       # stands for the ctypes struct (unpicklable)
    assert "_pk" not in copy.deepcopy(ff).__dict__
    torch.save(ff, io.BytesIO())


def test_forward_only_raises_on_grad_inputs():
    import torch
    import alphafold2_b200 as A
    blk = A.EvoformerBlock(dim=32, seq_len=8, heads=2, dim_head=16, attn_dropout=0., ff_dropout=0.)
    x = torch.randn(1, 8, 8, 32, requires_grad=True)
    m = torch.randn(1, 2, 8, 32)
    with pytest.raises(RuntimeError, match="forward-only"):
        blk((x, m, None, None))
    with pytest.raises(RuntimeError, match="forward-only"):
        A.FeedForward(dim=32)(x)


def test_cpu_tensor_raises():
    import torch
    import alphafold2_b200 as A
    ff = A.FeedForward(dim=32)
    with pytest.raises(RuntimeError):
        ff(torch.randn(2, 32))
