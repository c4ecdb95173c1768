"""Compare two builds of one translation unit kernel by kernel, at the SASS level.

    python tools/sass_diff.py OLD.o NEW.o [--ptxas OLD.txt NEW.txt]

Each kernel's instruction stream comes from `cuobjdump -sass`, keyed on its demangled name without the parameter
list, with the address column and the encoding comments dropped.  A kernel is IDENTICAL when the streams match,
PARAMS when they match once every constant-bank-0 offset (`c[0x0][...]`, the kernel parameters, also register- and
uniform-register-indexed) is masked, and DIFFERS otherwise.  --ptxas takes the `-Xptxas -v` logs of the two builds and adds each kernel's
registers and spill bytes to the report.  Needs cuobjdump and cu++filt (CUDA toolkit) on PATH or in
/usr/local/cuda/bin; no GPU.
"""
from __future__ import annotations

import argparse
import os
import re
import shutil
import subprocess
import sys


def _tool(name):
    return shutil.which(name) or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)


def _demangle(names):
    out = subprocess.run([_tool("cu++filt")], input="\n".join(names), capture_output=True, text=True, check=True)
    return dict(zip(names, out.stdout.splitlines()))


def _key(demangled):
    """'void ns::k<(bool)1, (int)64>(args)' -> 'ns::k<true, 64>'"""
    depth, i = 0, len(demangled)
    while i > 0:  # drop the parameter list: the last parenthesised group
        i -= 1
        depth += {")": 1, "(": -1}.get(demangled[i], 0)
        if depth == 0:
            break
    name = demangled[:i].replace("(bool)1", "true").replace("(bool)0", "false")
    name = re.sub(r"\(int\)(-?\d+)", r"\1", name)
    return name[5:] if name.startswith("void ") else name


def sass(obj):
    """{mangled name: [instruction text]} of every kernel in obj."""
    text = subprocess.run([_tool("cuobjdump"), "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(re.sub(r"\s+", " ", m.group(1)))
    return funcs


def ptxas(log):
    """{mangled name: (registers, spill store bytes, spill load bytes)} from an -Xptxas -v log; a field missing from a
    kernel's block stays None."""
    res, cur = {}, None
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            res[cur] = [None, None, None]
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            res[cur][1:] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            res[cur][0] = int(m.group(1))
    return {k: tuple(v) for k, v in res.items()}


def _keyed(funcs, regs):
    dem = _demangle(list(funcs))
    return {_key(dem[m]): (ins, regs.get(m)) for m, ins in funcs.items()}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--ptxas", nargs=2, metavar=("OLD_LOG", "NEW_LOG"))
    a = ap.parse_args(argv)
    regs_old, regs_new = (ptxas(a.ptxas[0]), ptxas(a.ptxas[1])) if a.ptxas else ({}, {})
    old = _keyed(sass(a.old), regs_old)
    new = _keyed(sass(a.new), regs_new)
    mask = lambda ins: [re.sub(r"c\[0x0\]\[(U?R\d+\+)?0x[0-9a-f]+\]", r"c[0x0][\1*]", i) for i in ins]  # noqa: E731
    counts = {}
    for k in sorted(set(old) | set(new)):
        if k not in old or k not in new:
            verdict = "ONLY_NEW" if k in new else "ONLY_OLD"
        elif old[k][0] == new[k][0]:
            verdict = "IDENTICAL"
        elif mask(old[k][0]) == mask(new[k][0]):
            verdict = "PARAMS"
        else:
            verdict = "DIFFERS"
        counts[verdict] = counts.get(verdict, 0) + 1
        n_old = len(old[k][0]) if k in old else "-"
        n_new = len(new[k][0]) if k in new else "-"
        r_old = old.get(k, (None, None))[1]
        r_new = new.get(k, (None, None))[1]
        regs = f"  regs/spill st/ld {r_old} -> {r_new}" if a.ptxas else ""
        print(f"{verdict:9s} {n_old:>5} -> {n_new:<5} {k}{regs}")
    print(" ".join(f"{v}={n}" for v, n in sorted(counts.items())))
    return 0 if set(counts) <= {"IDENTICAL", "PARAMS"} else 1


if __name__ == "__main__":
    sys.exit(main())
