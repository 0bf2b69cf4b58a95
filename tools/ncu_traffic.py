"""dram__bytes_read.sum + dram__bytes_write.sum of the first kernel in an .ncu-rep, as the JSON
entry profiles/ncu_traffic.json holds (bench.py copies it into roofline.traffic).
    python tools/ncu_traffic.py <capture>.ncu-rep [raw.csv]"""
import csv
import json
import subprocess
import sys

MULT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}


def from_rows(rows):
    if len(rows) < 3:
        return None
    h, units, r = rows[0], rows[1], rows[2]

    def get(k):
        if k not in h:
            return None
        i = h.index(k)
        return float(r[i].replace(",", "")) * MULT.get(units[i], 1.0)

    rd, wr = get("dram__bytes_read.sum"), get("dram__bytes_write.sum")
    return {"kernel": r[h.index("Kernel Name")] if "Kernel Name" in h else "",
            "read": rd, "write": wr, "bytes": (rd or 0.0) + (wr or 0.0)}


def main():
    if len(sys.argv) > 2:  # a raw csv exported earlier
        text = open(sys.argv[2]).read()
    else:
        text = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"],
                              capture_output=True, text=True).stdout
    print(json.dumps(from_rows(list(csv.reader(text.splitlines())))))


if __name__ == "__main__":
    main()
