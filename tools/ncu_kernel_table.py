"""Per-kernel evidence table from an `ncu --set full` report: duration, tensor-pipe %, DRAM traffic, achieved GB/s.

    python tools/ncu_kernel_table.py out/r02_zoo.ncu-rep [more.ncu-rep ...] > out/kernel_table.md

Tensor-pipe %: `sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg / (4 * sm__cycles_elapsed.avg)` — the counter
is the per-SM sum over the four tensor sub-pipes.
Durations under ncu are cold-cache at whatever clock the replay ran (column `GHz`); they are not bench numbers."""
import csv
import io
import subprocess
import sys

KEYS = {
    "dur": "gpu__time_duration.sum",
    "cyc": "sm__cycles_elapsed.avg",
    "hmma": "TPC.TriageCompute.sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg",
    "hmma2": "sm__pipe_tensor_subpipe_hmma_cycles_active_realtime.avg",
    "dr": "dram__bytes_read.sum",
    "dw": "dram__bytes_write.sum",
    "l2sm": "l1tex__m_xbar2l1tex_read_bytes.sum",
    "ghz": "sm__cycles_elapsed.avg.per_second",
    "regs": "launch__registers_per_thread",
    "smem": "launch__shared_mem_per_block_dynamic",
    "occ": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "dram_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
}
UNIT_SCALE = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6,
              "nsecond": 1e-3, "usecond": 1, "msecond": 1e3, "second": 1e6}


def rows_of(path):
    txt = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    r = list(csv.reader(io.StringIO(txt[txt.find('"ID"'):])))
    hdr, units = r[0], r[1]
    for row in r[2:]:
        d = dict(zip(hdr, row))
        u = dict(zip(hdr, units))
        yield d, u


def num(d, u, key):
    v = d.get(key, "")
    if v in ("", "n/a", "no data") or not v.replace(",", "").replace(".", "").replace("-", "").replace("e", "").replace("+", "").isdigit():
        return None
    unit = u.get(key, "").split("/")[0]
    return float(v.replace(",", "")) * UNIT_SCALE.get(unit, 1)


def main(paths):
    print("| kernel | grid | dur µs | GHz | tensor-pipe % | DRAM R+W MB | DRAM GB/s | DRAM % | L2→SM MB | regs | smem KB |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for p in paths:
        for d, u in rows_of(p):
            name = d.get("Kernel Name", "").replace("mgb::", "").replace("void ", "")
            name = name.split("(")[0]
            dur = num(d, u, KEYS["dur"])
            cyc = num(d, u, KEYS["cyc"])
            hm = num(d, u, KEYS["hmma"])
            if hm is None:
                hm = num(d, u, KEYS["hmma2"])
            tp = 100.0 * hm / (4 * cyc) if (hm is not None and cyc) else None
            dr, dw = num(d, u, KEYS["dr"]) or 0.0, num(d, u, KEYS["dw"]) or 0.0
            l2 = num(d, u, KEYS["l2sm"])
            ghz = num(d, u, KEYS["ghz"])
            f = lambda v, s="%.1f": ("-" if v is None else s % v)  # noqa: E731
            print(f"| {name} | {d.get('Grid Size', '')} | {f(dur)} | {f(ghz, '%.2f')} | {f(tp)} | {(dr + dw) / 1e6:.1f} | "
                  f"{(dr + dw) / dur / 1e3 if dur else 0:.0f} | {f(num(d, u, KEYS['dram_pct']))} | "
                  f"{f(l2 / 1e6 if l2 is not None else None)} | {d.get(KEYS['regs'], '')} | "
                  f"{f((num(d, u, KEYS['smem']) or 0) / 1024)} |")


if __name__ == "__main__":
    main(sys.argv[1:])
