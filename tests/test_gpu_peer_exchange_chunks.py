"""-m gpu: the chunk-table peer-store exchange (af2_peer_exchange_chunks, csrc/peer_api.inl) and PeerExchange over uneven
shards, with P ranks emulated in one process on one GPU (the method of tests/test_gpu_peer_exchange.py).

All P arenas live on the same device and share one table of arena bases; each rank's arena is laid out by
PeerExchange.layout for that rank (one offset table, every rank's own shapes).  The ranks run one after another on one
stream; before the first rank of an exchange is launched, every flag slot a correct kernel waits on is armed with e + 256
(e = the exchange's epoch), so each rank's wait passes at once; after the last rank every one of those slots must hold
exactly e again, stored by the rank it belongs to.

Checked after every exchange, on every arena, byte for byte: the destination buffers against the row / column shards of
the full tensors (shard_offsets), that every other byte (sources, padding, the other track) is unchanged, and the control
block (flags, epochs, completion counters, error word).  The destination buffer is refilled with a sentinel before each
exchange, so every byte it must hold has to be stored by the kernel."""
import ctypes as C

import pytest
import torch

from alphafold2_b200 import _lib
from alphafold2_b200.parallel import PeerExchange, _RawCuda, shard_offsets

pytestmark = pytest.mark.gpu

PAIR, MSA = PeerExchange.PAIR, PeerExchange.MSA
SENTINEL = 0xA5
CTRL = 4096
FLAGS, EPOCH, DONE, ERR = 0, 256, 272, 288   # control-block word indices: flags[2][32], epoch[2], done[2], err
DEV = torch.device("cuda", 0)

CASES = [                    # N, S, d, P
    (7, 3, 16, 2),           # 256 / 192 B rows: less than one segment of 16 KB
    (50, 7, 64, 3),          # 4352 / 4096 B rows, odd rank count
    (61, 1, 64, 8),          # S = 1: seven ranks have no MSA rows and send nothing in the MSA row -> column exchange
    (259, 18, 128, 4),       # 33280 / 32768 B rows: three and two segments
    (33, 40, 4, 32),         # 32 ranks, 32 / 16 B rows; one rank with two pair rows, every lane of the barrier warp
    (3, 131069, 4, 2),       # MSA chunks of 65535 and 65534 rows (the largest grid.y), 32 / 16 B rows
    (48, 16, 64, 8),         # an even shape through the chunk table
]
SEQUENCE = [("r2c", PAIR, 0), ("r2c", MSA, 1), ("c2r", PAIR, 0), ("c2r", MSA, 1), ("r2c", PAIR, 0), ("r2c", MSA, 0)]


class _Ranks:
    """P arenas, each laid out by PeerExchange.layout for its rank, the device table of their bases, and what every arena
    must hold."""

    def __init__(self, N, S, d, P, bases):
        self.N, self.S, self.d, self.P, self.bases = N, S, d, P, bases
        self.lays = [PeerExchange.layout(N, S, d, P, r) for r in range(P)]
        self.total = self.lays[0]["total"]
        self.mem = [torch.as_tensor(_RawCuda(b, self.total), device=DEV) for b in bases]
        assert all(a.data_ptr() == b for a, b in zip(self.mem, bases))
        self.table = torch.tensor(bases, dtype=torch.int64, device=DEV)
        for a in self.mem:
            assert not a[:CTRL].any(), "af2_peer_alloc must zero the control block"
            a[CTRL:] = SENTINEL
        self.expect = [a.clone() for a in self.mem]
        self.epoch = [0, 0]
        self.offsets = {PAIR: shard_offsets(N, P), MSA: shard_offsets(S, P)}

    def view(self, r, a, track, layout):
        o, shape = self.lays[r]["off"][(track, layout)], self.lays[r]["shapes"][(track, layout)]
        return a[o:o + shape[0] * shape[1] * shape[2] * 4].view(torch.int32).view(shape)

    def shard(self, full, track, layout, r):
        """Rank r's rows (layout "row") or columns ("col") of the full tensor of `track`."""
        if layout == "row":
            o = self.offsets[track]
            return full[o[r]:o[r + 1]]
        o = self.offsets[PAIR]
        return full[:, o[r]:o[r + 1]]

    def fill_rows(self, track, full):
        for r in range(self.P):
            for a in (self.mem[r], self.expect[r]):
                self.view(r, a, track, "row").copy_(self.shard(full, track, "row", r))

    def exchange(self, direction, track, channel, full, launch):
        P, dst_l = self.P, ("col" if direction == "r2c" else "row")
        e = self.epoch[channel] + 1
        for r in range(P):
            o = self.lays[r]["off"][(track, dst_l)]
            n = self.view(r, self.mem[r], track, dst_l).numel() * 4
            self.mem[r][o:o + n] = SENTINEL
            self.view(r, self.expect[r], track, dst_l).copy_(self.shard(full, track, dst_l, r))
            ctrl = self.expect[r][:CTRL].view(torch.int32)
            ctrl[FLAGS + 32 * channel:FLAGS + 32 * channel + P] = e
            ctrl[EPOCH + channel] = e
            ctrl[DONE + channel] = 0
            if P > 1:
                self.mem[r][:CTRL].view(torch.int32)[FLAGS + 32 * channel:FLAGS + 32 * channel + P] = e + 256
        for r in range(P):
            launch(r, direction, track, channel)
        self.epoch[channel] = e
        self.check(f"{direction} track {track} channel {channel} (epoch {e})")

    def check(self, what):
        torch.cuda.synchronize()
        lib = _lib.load()
        for r in range(self.P):
            got, want = self.mem[r], self.expect[r]
            if not torch.equal(got, want):
                bad = (got != want).nonzero().flatten()
                i = int(bad[0])
                raise AssertionError(f"{what}: arena {r} of {self.P}: {bad.numel()} bytes differ, the first at byte {i} "
                                     f"({self.where(r, i)}): {int(got[i]):#04x}, expected {int(want[i]):#04x}")
            assert lib.af2_peer_error(self.bases[r]) == 0, f"{what}: arena {r}: a barrier timed out"

    def where(self, r, byte):
        if byte < CTRL:
            w = byte // 4
            names = [(FLAGS, 64, "flags"), (EPOCH, 2, "epoch"), (DONE, 2, "done"), (ERR, 1, "err")]
            return next((f"{n}[{w - s}]" for s, k, n in names if s <= w < s + k), f"control word {w}")
        for (track, layout), o in self.lays[r]["off"].items():
            shape = self.lays[r]["shapes"][(track, layout)]
            if o <= byte < o + shape[0] * shape[1] * shape[2] * 4:
                return f"{('pair', 'msa')[track]} {layout} buffer + {byte - o}"
        return "padding"


@pytest.fixture
def ranks():
    """make(N, S, d, P) -> _Ranks over P fresh arenas; they are freed when the test ends."""
    lib = _lib.load()
    bases = []

    def make(N, S, d, P):
        total = PeerExchange.layout(N, S, d, P)["total"]
        for _ in range(P):
            b = C.c_void_p()
            _lib.check(lib.af2_peer_alloc(total, C.byref(b)))
            bases.append(b.value)
        return _Ranks(N, S, d, P, bases[-P:])

    yield make
    torch.cuda.synchronize()
    for b in bases:
        _lib.check(lib.af2_peer_free(b))


def _chunk_table(plan, dst_buffer_off, P):
    return (_lib.PeerChunk * P)(*[_lib.PeerChunk(c["src_off"], dst_buffer_off + c["dst_off"], c["dst_row_stride"], c["row_bytes"],
                                                 c["rows"], 0) for c in plan["chunks"]])


def _raw_launcher(rk):
    """Rank r's launch of af2_peer_exchange_chunks with the arguments of PeerExchange.plan_*_ragged."""
    lib = _lib.load()

    def launch(r, direction, track, channel):
        src_l, dst_l = ("row", "col") if direction == "r2c" else ("col", "row")
        plan = (PeerExchange.plan_rows_to_cols_ragged if direction == "r2c" else PeerExchange.plan_cols_to_rows_ragged)(
            rk.offsets[track], rk.offsets[PAIR], rk.d, r)
        src = rk.bases[r] + rk.lays[r]["off"][(track, src_l)]
        _lib.check(lib.af2_peer_exchange_chunks(src, plan["src_row_stride"], _chunk_table(plan, rk.lays[r]["off"][(track, dst_l)], rk.P),
                                                rk.table.data_ptr(), channel, r, rk.P, torch.cuda.current_stream().cuda_stream))
    return launch


def _run_sequence(rk, launch):
    full = {PAIR: torch.randint(-2 ** 31, 2 ** 31 - 1, (rk.N, rk.N, rk.d), dtype=torch.int32, device=DEV),
            MSA: torch.randint(-2 ** 31, 2 ** 31 - 1, (rk.S, rk.N, rk.d), dtype=torch.int32, device=DEV)}
    rk.fill_rows(PAIR, full[PAIR])
    rk.fill_rows(MSA, full[MSA])
    rk.check("initial state")
    for direction, track, channel in SEQUENCE:
        rk.exchange(direction, track, channel, full[track], launch)
    assert rk.epoch == [4, 2]


@pytest.mark.parametrize("N,S,d,P", CASES)
def test_chunk_exchange_kernel(ranks, N, S, d, P):
    torch.manual_seed(N * 131 + P)
    rk = ranks(N, S, d, P)
    _run_sequence(rk, _raw_launcher(rk))


@pytest.mark.parametrize("N,S,d,P", CASES)
def test_peer_exchange_class_uneven(ranks, N, S, d, P):
    """The same sequence through PeerExchange.rows_to_cols / cols_to_rows of P objects attached to one shared table, each
    with its rank's layout: the returned tensor is the rank's own destination buffer with its own shape."""
    torch.manual_seed(N * 131 + P + 1)
    rk = ranks(N, S, d, P)
    exs = [PeerExchange.attach(P, r, rk.bases[r], rk.table, DEV, rk.lays[r]) for r in range(P)]

    def launch(r, direction, track, channel):
        ex = exs[r]
        src_l, dst_l = ("row", "col") if direction == "r2c" else ("col", "row")
        fn = ex.rows_to_cols if direction == "r2c" else ex.cols_to_rows
        out = fn(ex.buffer(track, src_l), track, channel)
        assert tuple(out.shape) == rk.lays[r]["shapes"][(track, dst_l)]
        assert out.numel() == 0 or out.data_ptr() == rk.bases[r] + rk.lays[r]["off"][(track, dst_l)]

    _run_sequence(rk, launch)
    assert all(ex.exchanges == len(SEQUENCE) for ex in exs) and not any(ex.error() for ex in exs)


def test_rejected_chunk_arguments_write_nothing(ranks):
    """Each malformed call raises ValueError before anything is launched: no arena byte changes."""
    lib = _lib.load()
    P, N, S, d = 2, 3, 131069, 4
    rk = ranks(N, S, d, P)
    rk.fill_rows(MSA, torch.randint(-2 ** 31, 2 ** 31 - 1, (S, N, d), dtype=torch.int32, device=DEV))
    for a in rk.mem + rk.expect:             # a launch that should not have happened finds its barrier open at once
        a[:CTRL].view(torch.int32)[FLAGS:FLAGS + 64] = 1 << 20
    plan = PeerExchange.plan_rows_to_cols_ragged(rk.offsets[MSA], rk.offsets[PAIR], d, 0)
    good_chunks = [dict(c) for c in plan["chunks"]]
    assert [c["rows"] for c in good_chunks] == [65535, 65535] and [c["row_bytes"] for c in good_chunks] == [32, 16]
    dst_off = rk.lays[0]["off"][(MSA, "col")]
    good = dict(src=rk.bases[0] + rk.lays[0]["off"][(MSA, "row")], src_row_stride=plan["src_row_stride"], channel=0, rank=0, P=P)
    table33 = torch.tensor([rk.bases[i % P] for i in range(33)], dtype=torch.int64, device=DEV)

    def call(chunk_change=None, which=1, **change):
        a = {**good, **change}
        chunks = [dict(c) for c in good_chunks]
        if chunk_change:
            chunks[which].update(chunk_change)
        n = max(a["P"], 1)
        table = None if a.get("no_table") else _chunk_table(dict(chunks=(chunks * 33)[:n]), dst_off, n)
        return lib.af2_peer_exchange_chunks(a["src"], a["src_row_stride"], table, table33.data_ptr(), a["channel"], a["rank"],
                                            a["P"], torch.cuda.current_stream().cuda_stream)

    bad = [dict(chunk_change=dict(rows=65536)), dict(chunk_change=dict(rows=-1)), dict(chunk_change=dict(row_bytes=0)),
           dict(chunk_change=dict(row_bytes=8)), dict(chunk_change=dict(row_bytes=24)), dict(chunk_change=dict(row_bytes=-16)),
           dict(chunk_change=dict(src_off=8)), dict(chunk_change=dict(src_off=-16)), dict(chunk_change=dict(dst_off=8)),
           dict(chunk_change=dict(dst_row_stride=24)), dict(chunk_change=dict(dst_row_stride=-16)),
           dict(chunk_change=dict(rows=65536), which=0), dict(src_row_stride=plan["src_row_stride"] + 4), dict(src_row_stride=-16),
           dict(src=good["src"] + 8), dict(src=None), dict(P=0), dict(P=33), dict(rank=P), dict(rank=-1), dict(channel=2),
           dict(channel=-1), dict(no_table=True)]
    for change in bad:
        with pytest.raises(ValueError, match="peer_exchange_chunks"):
            _lib.check(call(**change))
        rk.check(f"rejected {change}")
