"""Compact per-launch table from an `ncu --page raw --csv` dump (run in the dev container, no GPU needed).
usage: python tools/summarize_ncu.py gpurun_out/prof_block_TAG_raw.csv profiles/TAG_block_C2_ncu_full_summary.csv [profiles/TAG_traffic.json]
The optional JSON holds, per bench.py kernel class, the average DRAM bytes per launch (dram__bytes_read.sum +
dram__bytes_write.sum) -- bench.py reports it as roofline.traffic."""
import csv
import json
import sys

WANT = [
    ("Kernel Name", "kernel"), ("Grid Size", "grid"), ("Block Size", "block"),
    ("gpu__time_duration.sum", "time_us"),
    ("dram__bytes_read.sum", "dram_read_MB"), ("dram__bytes_write.sum", "dram_write_MB"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "l2_pct"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pipe_pct"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_pct"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_active_pct"),
    ("launch__registers_per_thread", "regs"),
    ("launch__shared_mem_per_block_dynamic", "dyn_smem_KB"),
]


def kernel_class(name):
    if "proj_tc_kernel" in name:
        return "gemm_linear(wgmma)"
    if "gemm_tc_kernel" in name:
        return "gemm_per_channel(wgmma)" if name.rstrip(">").endswith(", 7") else "gemm_linear(wgmma)"
    if "attention_tc_kernel" in name:
        return "axial_attention(wgmma)"
    if "layernorm" in name or "pair_bias" in name:
        return "layernorm"
    if "chan_to_token" in name:
        return "channel_to_token"
    return "misc"


def to_bytes(v, unit):
    m = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}
    return float(v) * m.get(unit, 1)


def main(path, out_csv, out_json=None):
    rows = list(csv.reader(open(path)))
    hdr, units = rows[0], rows[1]
    cols = [(hdr.index(k), n, units[hdr.index(k)]) for k, n in WANT if k in hdr]
    ir, iw = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
    traffic = {}
    with open(out_csv, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(["launch"] + [(f"{n}[Mbyte]" if n.startswith("dram_") and n.endswith("_MB") else (f"{n}[us]" if n == "time_us" else (f"{n}[{u}]" if u else n))) for _, n, u in cols])
        for i, r in enumerate(rows[2:]):
            out = [i]
            name = r[hdr.index("Kernel Name")].split("(")[0].replace("void ", "")
            for c, n, u in cols:
                v = r[c]
                if n == "kernel":
                    v = name
                elif n.startswith("dram_") and n.endswith("_MB"):
                    v = f"{to_bytes(v, u) / 1e6:.3f}"          # ncu picks one unit per column and capture: normalise to MB
                elif n == "time_us":
                    v = f"{float(v) * {'ns': 1e-3, 'us': 1.0, 'ms': 1e3, 's': 1e6}.get(u, 1.0):.3f}"
                else:
                    try:
                        v = f"{float(v):.3f}".rstrip("0").rstrip(".")
                    except ValueError:
                        pass
                out.append(v)
            w.writerow(out)
            t = traffic.setdefault(kernel_class(name), [0, 0.0])
            t[0] += 1
            t[1] += to_bytes(r[ir], units[ir]) + to_bytes(r[iw], units[iw])
    if out_json:
        json.dump({k: {"launches": v[0], "dram_bytes_per_launch": v[1] / v[0]} for k, v in traffic.items()},
                  open(out_json, "w"), indent=1)


if __name__ == "__main__":
    main(*sys.argv[1:])
