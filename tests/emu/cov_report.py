#!/usr/bin/env python3
"""Reads the counters of a coverage build of the host emulation (tests/emu/build_cov.sh) and lists, for the F0 decision
kernels and their device helpers, the source lines that never ran and the branches that were never taken.

    python tests/emu/cov_report.py /tmp/cov

An instrument for whoever tests or rewrites these kernels, not a gate: lines compiled out of the emulation (#ifndef
WB_EMU) do not appear at all, and a branch gcov reports may be one the compiler made (a loop's entry test, the two
halves of a && condition)."""
import os
import re
import subprocess
import sys
import tempfile

FUNCTIONS = {
    "wb_harvest.cu": ["hv_min_rel_error", "harvest_remove_kernel", "hv_boundaries", "hv_select_best", "hv_extend",
                      "hv_search_score", "harvest_contour_kernel", "hv_filter_section", "harvest_smooth_kernel"],
    "wb_dio.cu": ["dio_select_best", "dio_contour_kernel"],
}


def function_spans(path, names):
    """{name: (first line, last line)} from the source text: the definition's line to its closing brace in column 0"""
    lines = open(path).read().split("\n")
    spans = {}
    for name in names:
        pat = re.compile(r"^(WB_DEV|WB_KERNEL\([^)]*\))\s.*\b" + name + r"\(")
        for i, ln in enumerate(lines):
            if pat.match(ln):
                j = i
                while lines[j] != "}":
                    j += 1
                spans[name] = (i + 1, j + 1)
                break
    return spans


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else "/tmp/cov")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "world_b200", "csrc")
    total_lines = total_branches = 0
    for fname, names in FUNCTIONS.items():
        stem = fname[:-3]
        if not os.path.exists(os.path.join(out, stem + ".gcda")):
            print(f"{fname}: no counters in {out} (run something through WB_EMU_LIB first)")
            continue
        with tempfile.TemporaryDirectory() as tmp:
            subprocess.check_call(["gcov", "-b", "-c", "-o", out, os.path.join(out, stem + ".o")], cwd=tmp,
                                  stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            text = open(os.path.join(tmp, fname + ".gcov")).read().split("\n")
        spans = function_spans(os.path.join(src, fname), names)
        missed_lines, missed_branches, executable = {}, {}, {}
        cur = None
        for ln in text:
            m = re.match(r"\s*([0-9#=\-*]+):\s*(\d+):(.*)", ln)
            if m:
                cur = int(m.group(2))
                count = m.group(1).rstrip("*")
                for name, (a, b) in spans.items():
                    if a <= cur <= b and count != "-":
                        executable[name] = executable.get(name, 0) + 1
                        if count.startswith("#") or count.startswith("="):
                            missed_lines.setdefault(name, []).append((cur, m.group(3).strip()))
                continue
            m = re.match(r"branch\s+(\d+) (never executed|taken (\d+))", ln)
            if m and cur is not None and (m.group(2) == "never executed" or m.group(3) == "0"):
                for name, (a, b) in spans.items():
                    if a <= cur <= b:
                        missed_branches.setdefault(name, []).append((cur, int(m.group(1))))
        for name in names:
            if name not in spans:
                print(f"{fname}: {name} not found")
                continue
            ml, mb = missed_lines.get(name, []), missed_branches.get(name, [])
            total_lines += len(ml)
            total_branches += len(mb)
            print(f"{fname} {name} (lines {spans[name][0]}-{spans[name][1]}): {executable.get(name, 0)} executable "
                  f"lines, {len(ml)} never ran, {len(mb)} branch outcomes never taken")
            for n, t in ml:
                print(f"    line {n} never ran: {t}")
            by_line = {}
            for n, b in mb:
                by_line.setdefault(n, []).append(b)
            for n in sorted(by_line):
                print(f"    line {n}: branch {', '.join(map(str, by_line[n]))} never taken")
    print(f"total: {total_lines} lines never ran, {total_branches} branch outcomes never taken")


if __name__ == "__main__":
    main()
