"""Summarise an `ncu --set full` capture of the tensor-core launches of one step: per-launch duration, DRAM bytes, tensor-pipe activity,
and the per-launch average DRAM traffic.
python tools/ncu_tensor_summary.py x.ncu-rep tensor_kernels.txt traffic.json "<command line>" """
import csv
import io
import json
import subprocess
import sys

rep, out_txt, out_json, cmd = sys.argv[1], sys.argv[2], sys.argv[3], sys.argv[4]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr = rows[0]


def col(name):
    return hdr.index(name)


def num(s):
    return float(s.replace(",", ""))


iname, igrid = col("Kernel Name"), col("Grid Size")
idur, ird, iwr = col("gpu__time_duration.sum"), col("dram__bytes_read.sum"), col("dram__bytes_write.sum")
units = rows[1]
tensor_cols = [i for i, h in enumerate(hdr) if h == "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"]  # chip-wide: small grids read low
scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
dscale = {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "nsecond": 1e-3}
lines, tot_rd, tot_wr, n = [], 0.0, 0.0, 0
for r in rows[2:]:
    if len(r) <= idur or not r[idur]:
        continue
    dur = num(r[idur]) * dscale.get(units[idur], 1.0)
    rd, wr = num(r[ird]) * scale.get(units[ird], 1.0), num(r[iwr]) * scale.get(units[iwr], 1.0)
    ta = max([num(r[i]) for i in tensor_cols if r[i] and r[i][0].isdigit()] or [0.0])
    name = r[iname].split("(")[0]
    lines.append(f"{n:2d} {name:46s} {dur:8.1f} us  dram_rd {rd / 1e6:8.1f} MB  dram_wr {wr / 1e6:8.1f} MB  tensor_active {ta:5.1f} %  grid {r[igrid].split(',')[0].strip('( ')}")
    tot_rd += rd
    tot_wr += wr
    n += 1
with open(out_txt, "w") as f:
    f.write(f"# ncu --set full, every tensor-core launch of one step, batch 256 x 3 s, bf16x3\n# command: {cmd}\n"
            "# per-launch times are cold-cache and serialised; DRAM bytes are per launch\n")
    f.write("\n".join(lines) + "\n")
    f.write(f"# {n} launches: dram read {tot_rd / 1e9:.3f} GB, write {tot_wr / 1e9:.3f} GB per step; average traffic per launch {(tot_rd + tot_wr) / n / 1e6:.1f} MB\n")
json.dump({"traffic_bytes_per_launch": (tot_rd + tot_wr) / n, "launches": n, "dram_read_bytes_per_step": tot_rd, "dram_write_bytes_per_step": tot_wr,
           "source": f"{out_txt} (ncu --set full, dram__bytes_read.sum + dram__bytes_write.sum averaged over the {n} tensor-core launches of one step)"},
          open(out_json, "w"), indent=1)
print(open(out_txt).read())
