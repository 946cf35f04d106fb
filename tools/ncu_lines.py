"""Per-source-line profile: joins an ncu report's per-SASS-instruction samples with nvdisasm line info.
usage: ncu_lines.py <report.ncu-rep> <kernel-substring> [top]   (the .so must be the build that was profiled)"""
import collections
import csv
import glob
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def line_table(kernel):
    tmp = tempfile.mkdtemp()
    subprocess.run(["cuobjdump", "-xelf", "all", os.path.join(ROOT, "world_b200", "lib", "libworld_b200.so")],
                   cwd=tmp, capture_output=True)
    for cub in glob.glob(os.path.join(tmp, "*sm_90a.cubin")):
        txt = subprocess.run(["nvdisasm", "--print-line-info", cub], capture_output=True, text=True).stdout
        m = re.search(r"\.text\.(\S*%s\S*):" % re.escape(kernel), txt)
        if not m:
            continue
        body = txt[m.end():]
        end = re.search(r"\n//-+ \.", body)
        body = body[:end.start()] if end else body
        table, cur = [], ("?", 0)
        for ln in body.splitlines():
            f = re.search(r'//## File "([^"]+)", line (\d+)', ln)
            if f:
                cur = (os.path.basename(f.group(1)), int(f.group(2)))
                continue
            if re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+\S", ln) and ".byte" not in ln and ".dword" not in ln:
                table.append(cur)
        return table
    raise SystemExit("kernel not found in the library")


def main(rep, kernel, top=30):
    table = line_table(kernel)
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout.splitlines()
    rows = list(csv.reader(out))
    hdr = rows[1]
    ni = hdr.index("Warp Stall Sampling (All Samples)"); ei = hdr.index("Instructions Executed")
    agg = collections.defaultdict(lambda: [0.0, 0.0])
    k = 0
    for r in rows[2:]:
        try:
            s, e = float(r[ni]), float(r[ei])
        except (ValueError, IndexError):
            continue
        key = table[k] if k < len(table) else ("?", -1)
        agg[key][0] += s; agg[key][1] += e
        k += 1
    ts = sum(v[0] for v in agg.values()); te = sum(v[1] for v in agg.values())
    print(f"# {rep} {kernel}: {k} SASS instructions, {len(table)} with line info; {ts:.0f} stall samples")
    src_cache = {}
    for (f, l), v in sorted(agg.items(), key=lambda kv: -kv[1][0])[:top]:
        path = os.path.join(ROOT, "world_b200", "csrc", f)
        if path not in src_cache:
            src_cache[path] = open(path).read().splitlines() if os.path.exists(path) else []
        text = src_cache[path][l - 1].strip()[:95] if 0 < l <= len(src_cache[path]) else ""
        print(f"stall {v[0] / ts:6.1%} inst {v[1] / te:6.1%}  {f}:{l:<4d} {text}")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], int(sys.argv[3]) if len(sys.argv) > 3 else 30)
