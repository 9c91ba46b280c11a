"""-m gpu: the peer-store exchange kernel (csrc/peer_api.inl) and PeerExchange (alphafold2_b200/parallel.py) with P ranks
emulated in one process on one GPU.

All P arenas live on the same device and share one table of arena bases, so rank r's launch stores its chunks into the
other ranks' arenas exactly as it does through the IPC mappings of a real run.  The ranks run one after another on one
stream and never meet in the barrier: before the first rank of an exchange is launched, every flag slot a correct kernel
waits on is armed with e + 256 (e = the exchange's epoch), so each rank's wait passes at once; after the last rank every
one of those slots must hold exactly e again, stored by the rank it belongs to.

Checked after every exchange, on every arena, byte for byte: the destination buffers against the all-to-all re-layout of
parallel.rows_to_cols / cols_to_rows, that every other byte (sources, padding, the other track) is unchanged, and the
control block (flags, epochs, completion counters, error word).  Not checked here, because it needs ranks that run at the
same time: the barrier's memory ordering between concurrent ranks and the IPC mappings (tests/parallel_check_multi_gpu.py
on several GPUs)."""
import ctypes as C

import pytest
import torch

from alphafold2_b200 import _lib
from alphafold2_b200.parallel import PeerExchange, _RawCuda

pytestmark = pytest.mark.gpu

PAIR, MSA = PeerExchange.PAIR, PeerExchange.MSA
SENTINEL = 0xA5                          # every arena byte beyond the control block that no exchange has written
CTRL = 4096
FLAGS, EPOCH, DONE, ERR = 0, 256, 272, 288   # control-block word indices: flags[2][32], epoch[2], done[2], err
DEV = torch.device("cuda", 0)

CASES = [                    # N, S, d, P; chunk rows are N/P * d * 4 bytes for both tracks
    (40, 8, 64, 1),          # one rank: its own flag store satisfies its wait, nothing is armed
    (136, 8, 256, 2),        # 69632 B rows: 4.25 segments of 16 KB (2.125 of 32 KB with 8 vectors per thread)
    (48, 12, 64, 3),         # odd rank count, 4096 B rows
    (256, 8, 256, 4),        # 65536 B rows: exactly 4 segments of 16 KB
    (48, 16, 64, 8),         # 1536 B rows: less than one segment
    (32, 32, 4, 32),         # 16 B rows (the minimum); every lane of the barrier warp and every flag slot
    (2, 131070, 4, 2),       # MSA track: 65535 rows of 16 B per chunk (the largest grid.y)
]
VARIANT_CASES = [(136, 8, 256, 2), (48, 16, 64, 8)]
# the schedule's pattern: each track alternates its two layouts; the MSA return runs on barrier channel 1 (_Deferred)
SEQUENCE = [("r2c", PAIR, 0), ("r2c", MSA, 1), ("c2r", PAIR, 0), ("c2r", MSA, 1), ("r2c", PAIR, 0), ("r2c", MSA, 0)]


def _rows_to_cols_ref(rows):
    """parallel.rows_to_cols on every rank at once: rank q's send chunk p goes to rank p, which stacks them in rank order."""
    P = len(rows)
    R, Cc, d = rows[0].shape
    send = [t.view(R, P, Cc // P, d).permute(1, 0, 2, 3) for t in rows]
    return [torch.stack([send[q][p] for q in range(P)]).reshape(P * R, Cc // P, d) for p in range(P)]


def _cols_to_rows_ref(cols):
    """parallel.cols_to_rows on every rank at once."""
    P = len(cols)
    RR, Cl, d = cols[0].shape
    send = [t.view(P, RR // P, Cl, d) for t in cols]
    return [torch.stack([send[q][p] for q in range(P)]).permute(1, 0, 2, 3).reshape(RR // P, P * Cl, d) for p in range(P)]


class _Ranks:
    """P arenas laid out by PeerExchange.layout, the device table of their bases, and what every arena must hold."""

    def __init__(self, P, lay, bases):
        self.P, self.lay, self.bases = P, lay, bases
        self.mem = [torch.as_tensor(_RawCuda(b, lay["total"]), device=DEV) for b in bases]
        assert all(a.data_ptr() == b for a, b in zip(self.mem, bases))
        self.table = torch.tensor(bases, dtype=torch.int64, device=DEV)
        for a in self.mem:
            assert not a[:CTRL].any(), "af2_peer_alloc must zero the control block"
            a[CTRL:] = SENTINEL
        self.expect = [a.clone() for a in self.mem]
        self.epoch = [0, 0]

    def view(self, a, track, layout):
        o, shape = self.lay["off"][(track, layout)], self.lay["shapes"][(track, layout)]
        return a[o:o + shape[0] * shape[1] * shape[2] * 4].view(torch.int32).view(shape)

    def fill_rows(self, track, full):
        """Rank r's row buffer of `track` = rows [r*R, (r+1)*R) of `full`."""
        R = full.shape[0] // self.P
        for r in range(self.P):
            for a in (self.mem[r], self.expect[r]):
                self.view(a, track, "row").copy_(full[r * R:(r + 1) * R])

    def exchange(self, direction, track, channel, launch):
        """One exchange: arm the barrier, launch rank 0..P-1, then compare every arena with what it must hold."""
        P, (src_l, dst_l) = self.P, (("row", "col") if direction == "r2c" else ("col", "row"))
        ref = (_rows_to_cols_ref if direction == "r2c" else _cols_to_rows_ref)([self.view(x, track, src_l) for x in self.expect])
        e = self.epoch[channel] + 1
        for r in range(P):
            o = self.lay["off"][(track, dst_l)]
            n = ref[r].numel() * 4
            self.mem[r][o:o + n] = SENTINEL                      # the kernel must write every destination byte
            self.view(self.expect[r], track, dst_l).copy_(ref[r])
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
                                     f"({self.where(i)}): {int(got[i]):#04x}, expected {int(want[i]):#04x}")
            assert lib.af2_peer_error(self.bases[r]) == 0, f"{what}: arena {r}: a barrier timed out"

    def where(self, byte):
        if byte < CTRL:
            w = byte // 4
            names = [(FLAGS, 64, "flags"), (EPOCH, 2, "epoch"), (DONE, 2, "done"), (ERR, 1, "err")]
            return next((f"{n}[{w - s}]" for s, k, n in names if s <= w < s + k), f"control word {w}")
        for (track, layout), o in self.lay["off"].items():
            shape = self.lay["shapes"][(track, layout)]
            if o <= byte < o + shape[0] * shape[1] * shape[2] * 4:
                return f"{('pair', 'msa')[track]} {layout} buffer + {byte - o}"
        return "padding"


@pytest.fixture
def ranks():
    """make(N, S, d, P) -> _Ranks over P fresh arenas; they are freed when the test ends."""
    lib = _lib.load()
    bases = []

    def make(N, S, d, P):
        lay = PeerExchange.layout(N, S, d, P)
        for _ in range(P):
            b = C.c_void_p()
            _lib.check(lib.af2_peer_alloc(lay["total"], C.byref(b)))
            bases.append(b.value)
        return _Ranks(P, lay, bases[-P:])

    yield make
    torch.cuda.synchronize()
    for b in bases:
        _lib.check(lib.af2_peer_free(b))


def _raw_launcher(rk):
    """Rank r's launch of af2_peer_exchange with the arguments of PeerExchange.plan_rows_to_cols / plan_cols_to_rows."""
    lib = _lib.load()

    def launch(r, direction, track, channel):
        src_l, dst_l = ("row", "col") if direction == "r2c" else ("col", "row")
        src = rk.view(rk.mem[r], track, src_l)
        plan = (PeerExchange.plan_rows_to_cols if direction == "r2c" else PeerExchange.plan_cols_to_rows)(*src.shape, rk.P, r)
        _lib.check(lib.af2_peer_exchange(src.data_ptr(), plan["src_peer_stride"], plan["src_row_stride"], rk.table.data_ptr(),
                                         rk.lay["off"][(track, dst_l)] + plan["dst_off"], plan["dst_row_stride"], plan["rows"],
                                         plan["row_bytes"], channel, r, rk.P, torch.cuda.current_stream().cuda_stream))
    return launch


def _run_sequence(rk, N, S, d, launch):
    pair = torch.randint(-2 ** 31, 2 ** 31 - 1, (N, N, d), dtype=torch.int32, device=DEV)
    msa = torch.randint(-2 ** 31, 2 ** 31 - 1, (S, N, d), dtype=torch.int32, device=DEV)
    rk.fill_rows(PAIR, pair)
    rk.fill_rows(MSA, msa)
    rk.check("initial state")
    for direction, track, channel in SEQUENCE:
        rk.exchange(direction, track, channel, launch)
        if direction == "c2r":                                   # the round trip returns the original row shards
            full = pair if track == PAIR else msa
            R = full.shape[0] // rk.P
            for r in range(rk.P):
                assert torch.equal(rk.view(rk.mem[r], track, "row"), full[r * R:(r + 1) * R]), ("round trip", track, r)
    assert rk.epoch == [4, 2]


@pytest.mark.parametrize("N,S,d,P", CASES)
def test_exchange_kernel(ranks, N, S, d, P):
    torch.manual_seed(N * 131 + P)
    rk = ranks(N, S, d, P)
    _run_sequence(rk, N, S, d, _raw_launcher(rk))


@pytest.mark.parametrize("variant", range(8))
@pytest.mark.parametrize("N,S,d,P", VARIANT_CASES)
def test_exchange_kernel_variants(ranks, monkeypatch, N, S, d, P, variant):
    """AF2_PEER_VARIANT (read on every call): bit 0 = 8 vectors per thread, bit 1 = one system fence per CTA instead of one
    per thread, bit 2 = destinations one after another instead of interleaved across CTAs."""
    monkeypatch.setenv("AF2_PEER_VARIANT", str(variant))
    torch.manual_seed(variant)
    rk = ranks(N, S, d, P)
    _run_sequence(rk, N, S, d, _raw_launcher(rk))


@pytest.mark.parametrize("N,S,d,P", CASES)
def test_peer_exchange_class(ranks, N, S, d, P):
    """The same sequence through PeerExchange.rows_to_cols / cols_to_rows of P objects attached to one shared table."""
    torch.manual_seed(N * 131 + P + 1)
    rk = ranks(N, S, d, P)
    exs = [PeerExchange.attach(P, r, rk.bases[r], rk.table, DEV, rk.lay) for r in range(P)]

    def launch(r, direction, track, channel):
        ex = exs[r]
        if direction == "r2c":
            out = ex.rows_to_cols(ex.buffer(track, "row"), track, channel)
            assert out.data_ptr() == rk.bases[r] + rk.lay["off"][(track, "col")]
        else:
            out = ex.cols_to_rows(ex.buffer(track, "col"), track, channel)
            assert out.data_ptr() == rk.bases[r] + rk.lay["off"][(track, "row")]
        assert tuple(out.shape) == rk.lay["shapes"][(track, "col" if direction == "r2c" else "row")]

    _run_sequence(rk, N, S, d, launch)
    assert all(ex.exchanges == len(SEQUENCE) for ex in exs) and not any(ex.error() for ex in exs)


def test_rejected_arguments_write_nothing(ranks):
    """Each malformed call raises ValueError before anything is launched: no arena byte changes."""
    lib = _lib.load()
    P = 2
    rk = ranks(2, 65535 * P, 4, P)
    msa = torch.randint(-2 ** 31, 2 ** 31 - 1, (65535 * P, 2, 4), dtype=torch.int32, device=DEV)
    rk.fill_rows(MSA, msa)
    for a in rk.mem + rk.expect:             # a launch that should not have happened finds its barrier open at once
        a[:CTRL].view(torch.int32)[FLAGS:FLAGS + 64] = 1 << 20
    table = torch.tensor([rk.bases[i % P] for i in range(33)], dtype=torch.int64, device=DEV)
    src = rk.view(rk.mem[0], MSA, "row")
    plan = PeerExchange.plan_rows_to_cols(*src.shape, P, 0)
    good = dict(src=src.data_ptr(), src_peer_stride=plan["src_peer_stride"], src_row_stride=plan["src_row_stride"],
                dst_off=rk.lay["off"][(MSA, "col")] + plan["dst_off"], dst_row_stride=plan["dst_row_stride"],
                rows=plan["rows"], row_bytes=plan["row_bytes"], channel=0, rank=0, P=P)
    assert good["rows"] == 65535 and good["row_bytes"] == 16
    bad = [dict(row_bytes=0), dict(row_bytes=8), dict(row_bytes=24), dict(src_peer_stride=good["src_peer_stride"] + 8),
           dict(src_row_stride=good["src_row_stride"] + 4), dict(dst_off=good["dst_off"] + 8),
           dict(dst_row_stride=good["dst_row_stride"] + 8), dict(src=good["src"] + 8), dict(P=0), dict(P=33),
           dict(rank=P), dict(rank=-1), dict(channel=2), dict(channel=-1), dict(rows=65536), dict(rows=0)]
    for change in bad:
        a = {**good, **change}
        with pytest.raises(ValueError, match="peer_exchange"):
            _lib.check(lib.af2_peer_exchange(a["src"], a["src_peer_stride"], a["src_row_stride"], table.data_ptr(), a["dst_off"],
                                             a["dst_row_stride"], a["rows"], a["row_bytes"], a["channel"], a["rank"], a["P"],
                                             torch.cuda.current_stream().cuda_stream))
        rk.check(f"rejected {change}")
