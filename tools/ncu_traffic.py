"""profiles/rNN_ncu_traffic.json from an `ncu --set full` capture of the dominant decode kernel (the gate/up GEMV launch made
by tools/ncu_gemv.py): dram__bytes_read.sum + dram__bytes_write.sum per launch next to the algorithmic bytes of that launch.
bench.py multiplies the algorithmic bytes of a decode step by this measured ratio for `roofline.traffic`.

  ncu --set full --clock-control none -k regex:gemv_tma -s 3 -c 2 -o gemv_gateup python tools/ncu_gemv.py
  python tools/ncu_traffic.py gemv_gateup.ncu-rep 35840 6656 > profiles/r02_ncu_traffic.json
"""
import csv
import json
import subprocess
import sys


def main():
    rep, N, K = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr = rows[0]
    col = {h: i for i, h in enumerate(hdr)}
    rd, wr, dur, names = [], [], [], []
    for r in rows[2:]:
        if len(r) < len(hdr):
            continue
        names.append(r[col["Kernel Name"]])
        scale = lambda v, unit: float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        rd.append(scale(r[col["dram__bytes_read.sum"]], rows[1][col["dram__bytes_read.sum"]]))
        wr.append(scale(r[col["dram__bytes_write.sum"]], rows[1][col["dram__bytes_write.sum"]]))
        dur.append(float(r[col["gpu__time_duration.sum"]]))
    n = len(rd)
    json.dump({"kernel": names[0] if names else None, "launches": n, "dram_bytes_per_launch": (sum(rd) + sum(wr)) / n,
               "dram_read_bytes_per_launch": sum(rd) / n, "dram_write_bytes_per_launch": sum(wr) / n,
               "algorithmic_bytes_per_launch": N * K * 2, "duration_us_cold_cache": sum(dur) / n,
               "source": rep, "shape": [N, K]}, sys.stdout, indent=1)
    print()


if __name__ == "__main__":
    main()
