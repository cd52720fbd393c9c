"""Extract the DRAM traffic of one kernel launch from an .ncu-rep (`ncu --set full`) into a JSON
file.  usage: ncu_traffic.py <report.ncu-rep> <kernel substring> <envs> <out.json>"""
import csv
import json
import subprocess
import sys

SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def main(path, kernel, envs, out):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        if kernel in r[hdr.index("Kernel Name")]:
            def val(k):
                i = hdr.index(k)
                return float(r[i].replace(",", "")) * SCALE.get(units[i], 1.0)
            d = {"kernel": r[hdr.index("Kernel Name")].split("(")[0], "envs": int(envs), "dram_bytes_read": val("dram__bytes_read.sum"),
                 "dram_bytes_write": val("dram__bytes_write.sum"), "gpu_time_us_under_ncu": float(r[hdr.index("gpu__time_duration.sum")]),
                 "source": path.split("/")[-1], "note": "ncu --set full --clock-control none, one launch, cold L2"}
            json.dump(d, open(out, "w"), indent=1)
            print(json.dumps(d))
            return
    raise SystemExit(f"no kernel matching {kernel!r} in {path}")


if __name__ == "__main__":
    main(*sys.argv[1:5])
