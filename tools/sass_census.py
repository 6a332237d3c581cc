"""SASS evidence for the sm_90a kernels: per-kernel mnemonic census + key-instruction extracts.

    python -m tools.sass_census [--so relora_b200/_C.so] --out DIR

Runs ``cuobjdump -sass`` on the built extension (no GPU needed), splits the listing per kernel and writes

* ``SASS_SUMMARY.md``                     one row per kernel: instruction count and the Hopper-path mnemonics
                                           (``HGMMA``/``QGMMA`` = bf16 / fp8 wgmma, ``UTMALDG``/``UTMASTG`` = TMA, ``UBLKCP`` = bulk copy,
                                           ``LDGMC``/``REDGMC`` = multimem, ``HMMA`` = legacy mma.sync), and ``gsb0``: the wgmma
                                           that close a batch (one per batch when ptxas batches, one per wgmma when it serialises);
* ``<kernel>.key.sass``                   every line of that kernel carrying one of those mnemonics (with its address), in order —
                                           the complete tensor-core / TMA / multimem instruction stream, not a truncated listing.

The census is what the "does it really use wgmma" question needs; full listings are reproducible with the command in the header
of each extract.
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY_RE = re.compile(r"\b(UTMA[A-Z]+[.\w]*|UBLKCP[.\w]*|LDGMC[.\w]*|STGMC[.\w]*|REDGMC[.\w]*|HMMA[.\w]*|HGMMA[.\w]*|QGMMA[.\w]*)")


def demangle(names):
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
        return dict(zip(names, out))
    except Exception:
        return {n: n for n in names}


def short(name: str) -> str:
    s = name.replace("(anonymous namespace)::", "").replace("rb::", "")
    s = re.sub(r"\(.*$", "", s)                  # drop the parameter list
    s = re.sub(r"^void\s+", "", s)
    return s


def listings(so: str) -> "OrderedDict[str, list]":
    """{mangled kernel name: its SASS lines} of ``cuobjdump -sass so``."""
    res = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"cuobjdump failed: {res.stderr[:500]}")
    kernels: "OrderedDict[str, list]" = OrderedDict()
    cur = None
    for line in res.stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
            continue
        if cur is not None and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            kernels[cur].append(line.rstrip())
    return kernels


def count(lines) -> "tuple[Counter, list]":
    """Mnemonic counts of one kernel's SASS lines, and the lines that carry a key mnemonic."""
    cnt = Counter()
    key_lines = []
    for ln in lines:
        m = KEY_RE.search(ln)
        if m:
            op = m.group(1)
            base = op.split(".")[0]
            cnt[base] += 1
            key_lines.append(ln)
            if base in ("HGMMA", "QGMMA") and "gsb0" in ln:
                cnt["gsb0"] += 1    # the wgmma that closes a batch: the warpgroup can wait for it
        if "MUFU.EX2" in ln:
            cnt["MUFU.EX2"] += 1
        if "BRA.U.ANY" in ln:
            cnt["waterfall"] += 1   # ELECT / R2UR / BRA.U.ANY loop around an instruction with uniform-register operands
    return cnt, key_lines


def census(so: str) -> "dict[str, Counter]":
    """{short demangled kernel name: mnemonic counts} of the built extension."""
    kernels = listings(so)
    names = demangle(list(kernels))
    return {short(names[k]): count(lines)[0] for k, lines in kernels.items()}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--so", default=os.path.join(ROOT, "relora_b200", "_C.so"))
    ap.add_argument("--out", required=True)
    a = ap.parse_args(argv)
    try:
        kernels = listings(a.so)
    except RuntimeError as e:
        sys.exit(str(e))
    names = demangle(list(kernels))
    os.makedirs(a.out, exist_ok=True)
    rows = []
    total = Counter()
    for mangled, lines in kernels.items():
        cnt, key_lines = count(lines)
        total.update(cnt)
        nm = short(names[mangled])
        rows.append((nm, len(lines), cnt))
        if key_lines:
            fn = re.sub(r"[^A-Za-z0-9_]+", "_", nm)[:120].strip("_") + ".key.sass"
            with open(os.path.join(a.out, fn), "w") as f:
                f.write(f"// {names[mangled]}\n// {len(lines)} SASS instructions; lines with wgmma / TMA / multimem mnemonics only\n"
                        f"// full listing: cuobjdump -sass -fun '{mangled}' relora_b200/_C.so\n")
                f.write("\n".join(key_lines) + "\n")
    cols = ["HGMMA", "QGMMA", "gsb0", "UTMALDG", "UTMASTG", "UBLKCP", "LDGMC", "REDGMC", "HMMA", "waterfall"]
    with open(os.path.join(a.out, "SASS_SUMMARY.md"), "w") as f:
        f.write("# SASS census of `relora_b200/_C.so` (sm_90a) — generated by `python -m tools.sass_census`\n\n")
        f.write("`HGMMA` / `QGMMA` = `wgmma.mma_async` with bf16 / fp8 operands; `UTMALDG`/`UTMASTG` = TMA load / store; `UBLKCP` = "
                "`cp.async.bulk`; `LDGMC`/`REDGMC` = `multimem.ld_reduce`/`red` (`multimem.st` has no mnemonic of its own: it is printed "
                "as `STG.E.128.STRONG.SYS` on the multicast address); `gsb0` = wgmma that close a batch (equal to HGMMA + QGMMA when "
                "ptxas serialises every wgmma); `HMMA` = legacy `mma.sync` (must be 0); `waterfall` = `BRA.U.ANY` "
                "count: ELECT / R2UR / branch loops ptxas wraps around instructions whose operands it cannot prove warp-uniform.\n\n")
        f.write("| kernel | SASS instr | " + " | ".join(cols) + " |\n|---|---|" + "---|" * len(cols) + "\n")
        for nm, n, cnt in sorted(rows, key=lambda r: -sum(r[2].values())):
            if not any(cnt.get(c, 0) for c in cols):
                continue
            f.write(f"| `{nm[:110]}` | {n} | " + " | ".join(str(cnt.get(c, 0)) for c in cols) + " |\n")
        f.write("\n**Totals**: " + ", ".join(f"{c} {total.get(c, 0)}" for c in cols) + f"; kernels: {len(kernels)}\n")
    print(f"{len(kernels)} kernels; totals: " + ", ".join(f"{c}={total.get(c, 0)}" for c in cols))


if __name__ == "__main__":
    main()
