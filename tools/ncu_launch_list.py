"""ncu CSV (--metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv) ->
the launch list of ONE step: the last `n` gcb:: launches, one line each
(id,kernel,gpu_time_ns,dram_read_bytes,dram_write_bytes), as bench.py's `ncu_traffic` reads it.

  python tools/ncu_launch_list.py ncu_raw.csv 61 "comment" > launches_ncu.csv
"""
import csv
import sys

path, n, comment = sys.argv[1], int(sys.argv[2]), (sys.argv[3] if len(sys.argv) > 3 else "")
rows = {}
with open(path, newline="") as f:
  lines = [l for l in f if not l.startswith("==")]
for r in csv.DictReader(lines):
  name = r.get("Kernel Name", "")
  if not any(k in name for k in ("mlp_chain_tc_kernel", "mlp_layer_tc_kernel", "mlp_layer_simt_kernel",
                                  "segment_sum_kernel", "pack_grid", "unpack_grid", "rows_to_image_kernel",
                                  "gather_rows_kernel", "tisr_kernel")):
    continue
  k = int(r["ID"])
  d = rows.setdefault(k, {"name": name})
  val = float(r["Metric Value"].replace(",", ""))
  unit = r.get("Metric Unit", "")
  m = r["Metric Name"]
  if m == "gpu__time_duration.sum":
    d["ns"] = val * {"ns": 1, "us": 1e3, "usecond": 1e3, "ms": 1e6, "msecond": 1e6, "nsecond": 1, "second": 1e9}.get(unit, 1)
  else:
    scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "KB": 1e3, "MB": 1e6, "GB": 1e9}.get(unit, 1)
    d["rd" if "read" in m else "wr"] = val * scale
ids = sorted(rows)[-n:]
print(f"# {comment}")
print("id,kernel,gpu_time_ns,dram_read_bytes,dram_write_bytes")
tot = [0.0, 0.0, 0.0]
for k in ids:
  d = rows[k]
  print(f"{k},{d['name']},{d.get('ns', 0):.0f},{d.get('rd', 0):.0f},{d.get('wr', 0):.0f}")
  tot[0] += d.get("ns", 0); tot[1] += d.get("rd", 0); tot[2] += d.get("wr", 0)
print(f"# total: {tot[0] / 1e6:.2f} ms serialised, {tot[1] / 1e9:.1f} GB read, {tot[2] / 1e9:.1f} GB written", file=sys.stderr)
