"""`ncu --csv --metrics ...` log (long format: one line per kernel launch and metric) -> one line per launch.

    python tools/ncu_long_summary.py ncu_log.csv summary.csv
"""
import csv
import sys

src, dst = sys.argv[1], sys.argv[2]
rows = {}
order = []
metrics = []
with open(src) as f:
    lines = [ln for ln in f if ln.startswith('"')]
for r in csv.DictReader(lines):
    key = r["ID"]
    if key not in rows:
        rows[key] = {"id": key, "kernel": r["Kernel Name"][:60], "grid": r["Grid Size"], "block": r["Block Size"]}
        order.append(key)
    name = f'{r["Metric Name"]} [{r["Metric Unit"]}]'
    if name not in metrics:
        metrics.append(name)
    rows[key][name] = r["Metric Value"].replace(",", "")
with open(dst, "w", newline="") as f:
    w = csv.DictWriter(f, fieldnames=["id", "kernel", "grid", "block"] + metrics)
    w.writeheader()
    for k in order:
        w.writerow(rows[k])
print("wrote", dst, len(order), "launches")
