"""Summarise Nsight Compute reports (.ncu-rep, `--set full`) into one JSON summary.

    python tools/ncu_summarise.py a.ncu-rep [b.ncu-rep ...] --out summary.json [--note "..."]

Per kernel NAME (launches of the same kernel are averaged, min/max duration kept): duration, DRAM bytes read + written and
the achieved DRAM GB/s against the measured copy bandwidth of MEASURED_PEAKS.json, L2 / L1 throughput %, tensor-pipe %,
warps active %, registers, grid/block, instruction-issue IPC and the four largest warp-stall reasons per issued instruction.
Reads the raw page through `ncu -i ... --page raw --csv` (ncu is in the build container; no GPU needed).
"""
import argparse
import csv
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3,
        "usecond": 1e-3, "msecond": 1.0, "nsecond": 1e-6, "second": 1e3}


def rows_of(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    r = list(csv.reader(io.StringIO(out)))
    hdr, units = r[0], r[1]
    return hdr, units, r[2:]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("reports", nargs="+")
    ap.add_argument("--out", required=True)
    ap.add_argument("--note", default="")
    a = ap.parse_args()
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    hbm = peaks.get("hbm_gbs", 6650.0)
    agg = {}
    for path in a.reports:
        hdr, units, rows = rows_of(path)
        col = {h: i for i, h in enumerate(hdr)}

        def val(row, name, scale=True):
            i = col.get(name)
            if i is None or row[i] in ("", "n/a"):
                return None
            v = float(row[i].replace(",", ""))
            return v * UNIT.get(units[i], 1.0) if scale else v

        for row in rows:
            name = row[col["Kernel Name"]]
            short = name.split("(")[0].replace("void ", "").replace("<unnamed>::", "").strip()
            d = agg.setdefault(short, {"launches": 0, "ms": [], "dram": [], "fields": {}})
            d["launches"] += 1
            ms = val(row, "gpu__time_duration.sum")
            d["ms"].append(ms)
            rd, wr = val(row, "dram__bytes_read.sum") or 0.0, val(row, "dram__bytes_write.sum") or 0.0
            d["dram"].append(rd + wr)
            f = d["fields"]
            for key, metric in (("tensor_pipe_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"),
                                ("l2_throughput_pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
                                ("l1_throughput_pct", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed"),
                                ("dram_throughput_pct", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
                                ("warps_active_pct", "sm__warps_active.avg.pct_of_peak_sustained_active"),
                                ("l2_hit_rate_pct", "lts__t_sector_hit_rate.pct"),
                                ("ipc_per_sm", "sm__inst_executed.avg.per_cycle_active"),
                                ("registers_per_thread", "launch__registers_per_thread"),
                                ("grid", "launch__grid_size"), ("block", "launch__block_size"),
                                ("l2_to_sm_bytes", "l1tex__m_xbar2l1tex_read_bytes.sum")):
                v = val(row, metric, scale=key == "l2_to_sm_bytes")
                if v is not None:
                    f.setdefault(key, []).append(v)
            stalls = {h.split("issue_stalled_")[1].split("_per_issue")[0]: float(row[i] or 0)
                      for h, i in col.items() if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")}
            d.setdefault("stalls", []).append(stalls)
    kernels = []
    for name, d in sorted(agg.items(), key=lambda kv: -sum(kv[1]["ms"])):
        n = d["launches"]
        ms = sum(d["ms"]) / n
        dram = sum(d["dram"]) / n
        k = {"kernel": name, "launches_profiled": n, "ms_avg": round(ms, 4), "ms_min": round(min(d["ms"]), 4), "ms_max": round(max(d["ms"]), 4),
             "dram_bytes_per_launch": round(dram), "dram_GBs": round(dram / ms / 1e6, 1), "dram_frac_of_measured_hbm": round(dram / ms / 1e6 / hbm, 4)}
        for key, vs in d["fields"].items():
            k[key] = round(sum(vs) / len(vs), 2)
        st = {}
        for s in d["stalls"]:
            for kk, v in s.items():
                st[kk] = st.get(kk, 0.0) + v / n
        k["top_stalls_per_issue"] = {kk: round(v, 2) for kk, v in sorted(st.items(), key=lambda kv: -kv[1])[:4]}
        kernels.append(k)
    json.dump({"reports": [os.path.basename(p) for p in a.reports], "note": a.note, "hbm_peak_GBs_measured": hbm,
               "how": "ncu --set full --clock-control none; per-launch values averaged per kernel name; cold caches, serialised",
               "kernels": kernels}, open(a.out, "w"), indent=1)
    for k in kernels[:30]:
        print(f"{k['kernel'][:60]:60s} {k['ms_avg']:8.4f} ms  dram {k['dram_GBs']:8.1f} GB/s ({k['dram_frac_of_measured_hbm']:.3f})  tensor {k.get('tensor_pipe_pct', 0):5.1f}%  L2 {k.get('l2_throughput_pct', 0):5.1f}%")


if __name__ == "__main__":
    main()
