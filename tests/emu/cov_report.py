#!/usr/bin/env python3
"""Reads the counters of a coverage build of the host emulation (tests/emu/build_cov.sh) and lists, for the F0 decision
kernels and their device helpers, the source lines that never ran and the branches that were never taken.

    python tests/emu/cov_report.py /tmp/cov
    python tests/emu/cov_report.py /tmp/cov wb_stonemask.cu:stonemask_kernel,sm_fix_f0 wb_spectral.cuh:dc_correction

Without FILE:FUNCTION,... arguments it reports on the F0 decision kernels below.  A header's functions are compiled
into every object that includes it: their counters are merged by source line (a line ran if it ran in any object) and
by instantiation and branch (a template instantiation's branch was taken if it was taken in any object).

An instrument for whoever tests or rewrites these kernels, not a gate: lines compiled out of the emulation (#ifndef
WB_EMU) do not appear at all, and a branch gcov reports may be one the compiler made (a loop's entry test, the two
halves of a && condition)."""
import glob
import gzip
import json
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


def requested(args):
    """FILE:FUNCTION,... arguments -> {file: [functions]}; none: FUNCTIONS"""
    if not args:
        return FUNCTIONS
    req = {}
    for a in args:
        fname, _, names = a.partition(":")
        if not names:
            sys.exit(f"{a}: expected FILE:FUNCTION[,FUNCTION...]")
        req.setdefault(fname, []).extend(names.split(","))
    return req


def counters(out, fname):
    """The merged counters of source file fname over its own object (a .cu) or every object (a header):
    ({line: count}, {(line, instantiation, branch index): count}), or None if no object has counters for it"""
    stems = [fname[:-3]] if fname.endswith(".cu") else sorted(f[:-5] for f in os.listdir(out) if f.endswith(".gcda"))
    lines, branches, found = {}, {}, False
    for stem in stems:
        if not os.path.exists(os.path.join(out, stem + ".gcda")):
            continue
        with tempfile.TemporaryDirectory() as tmp:
            subprocess.check_call(["gcov", "--json-format", "-b", "-c", "-o", out, os.path.join(out, stem + ".o")],
                                  cwd=tmp, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
            data = [json.load(gzip.open(f)) for f in glob.glob(os.path.join(tmp, "*.gcov.json.gz"))]
        for d in data:
            for entry in d["files"]:
                if os.path.basename(entry["file"]) != fname:
                    continue
                found = True
                names = {f["name"]: f["demangled_name"] for f in entry["functions"]}
                for ln in entry["lines"]:
                    n = ln["line_number"]
                    lines[n] = lines.get(n, 0) + ln["count"]
                    inst = names.get(ln.get("function_name", ""), ln.get("function_name", ""))
                    for k, b in enumerate(ln["branches"]):
                        key = (n, inst, k)
                        branches[key] = branches.get(key, 0) + b["count"]
    return (lines, branches) if found else None


def main():
    out = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else "/tmp/cov")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "world_b200", "csrc")
    total_lines = total_branches = 0
    for fname, names in requested(sys.argv[2:]).items():
        got = counters(out, fname)
        if got is None:
            print(f"{fname}: no counters in {out} (run something through WB_EMU_LIB first)")
            continue
        lines, branches = got
        text = open(os.path.join(src, fname)).read().split("\n")
        spans = function_spans(os.path.join(src, fname), names)
        for name in names:
            if name not in spans:
                print(f"{fname}: {name} not found")
                continue
            a, b = spans[name]
            executable = sorted(n for n in lines if a <= n <= b)
            ml = [n for n in executable if lines[n] == 0]
            mb = {}
            for (n, inst, k), c in sorted(branches.items()):
                if a <= n <= b and c == 0:
                    mb.setdefault((n, inst), []).append(k)
            n_mb = sum(len(v) for v in mb.values())
            total_lines += len(ml)
            total_branches += n_mb
            print(f"{fname} {name} (lines {a}-{b}): {len(executable)} executable lines, {len(ml)} never ran, "
                  f"{n_mb} branch outcomes never taken")
            for n in ml:
                print(f"    line {n} never ran: {text[n - 1].strip()}")
            for (n, inst), ks in sorted(mb.items()):
                print(f"    line {n}: branch {', '.join(map(str, ks))} never taken" + (f" in {inst}" if inst else ""))
    print(f"total: {total_lines} lines never ran, {total_branches} branch outcomes never taken")


if __name__ == "__main__":
    main()
