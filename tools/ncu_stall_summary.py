"""Warp-state sampling summary of ONE kernel launch of an ncu report captured with --set full --import-source on.

    python tools/ncu_stall_summary.py gpurun_out/gemm_pair_r2.ncu-rep [launch_index] [top_n]

Prints the stall-reason totals and the most sampled SASS instructions (address suffix, samples, executions, top stall reason).
Used to find what the producer / MMA / epilogue warps of the tensor-core kernels wait on."""
import csv
import io
import subprocess
import sys


def load(rep, launch):
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv", "--launch-skip", str(launch), "--launch-count", "1"],
                         capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    name = rows[0][1] if rows and len(rows[0]) > 1 else "?"
    hdr = rows[1]
    ia, isrc, isamp, iex = hdr.index("Address"), hdr.index("Source"), hdr.index("# Samples"), hdr.index("Instructions Executed")
    stall = [i for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
    seen, lst = set(), []
    for r in rows[2:]:
        if len(r) <= iex or not r[ia].startswith("0x") or r[ia] in seen:
            continue
        seen.add(r[ia])
        lst.append(r)
    return name, hdr, lst, (ia, isrc, isamp, iex), stall


def main():
    rep = sys.argv[1]
    launch = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    top_n = int(sys.argv[3]) if len(sys.argv) > 3 else 40
    name, hdr, lst, (ia, isrc, isamp, iex), stall = load(rep, launch)
    num = lambda s: int(s) if s.isdigit() else 0
    total = sum(num(r[isamp]) for r in lst)
    print(f"# {name}")
    print(f"# launch {launch}: {len(lst)} SASS instructions, {total} warp samples")
    agg = {}
    for r in lst:
        for i in stall:
            agg[hdr[i]] = agg.get(hdr[i], 0) + num(r[i])
    print("# stall totals: " + ", ".join(f"{k[6:]} {v}" for k, v in sorted(agg.items(), key=lambda kv: -kv[1])[:10]))
    for r in sorted(lst, key=lambda r: -num(r[isamp]))[:top_n]:
        st = max(((num(r[i]), hdr[i][6:]) for i in stall), default=(0, ""))
        print(f"{r[ia][-5:]} {num(r[isamp]):5d} x{num(r[iex]):7d}  {r[isrc].strip()[:84]:84s} {st[1]} {st[0]}")


if __name__ == "__main__":
    main()
