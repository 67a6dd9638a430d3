#!/usr/bin/env python
"""tools/sass_compare.py OLD NEW — compare the SASS of every kernel of two builds (cubins or liblmpc_b200.so).

Kernels are matched by variant and (N, M) across their old and new names:
  uniform  ftocp_kernel<N, M, 2, 4>  or  ftocp_kernel<N, M, 2, 4, false>
  sets     ftocp_sets_kernel<N, M, 2, 4>  or  ftocp_kernel<N, M, 2, 4, true>
and the other kernels of a step and of the lap books, each matched by its name with or without a template argument list of up
to five `false` flags, so that the instantiation without a per-controller table of an older build meets the untemplated kernel:
  default  knn_ltv_regress_kernel, ss_select_kernel, shift_state_kernel (<false>: no shape or lap-count table),
           books_refresh_kernel, commit_laps_books_kernel, seed_books_kernel, pool_import_kernel, pool_local_best_kernel,
           pool_export_kernel, commit_laps_kernel, seed_from_record_kernel and measure_kernel (untemplated; older builds had one
           flag per table they read: lap counts, lap reports, lap windows, lane rules, lane margins, lap schedules),
           sim_step_kernel and nominal_model_kernel (<false>: no surface table; older builds: <false, false> or
           <false, false, false>, no lap reports, no lap schedule and no surface table), observe_kernel (<false, false>: no
           observer prior table; older builds: <false> or untemplated)
  reports  sim_step_kernel<true, false> or <true, false, false> of an older build: lap reports, no lap schedule and no surface
           table (later builds have no such kernel: their sim_step_kernel<true> is the surface instantiation)
  surface  sim_step_kernel<true> and nominal_model_kernel<true>: the surface instantiations (builds with track surfaces)
  prior    observe_kernel<true, false> or <true>: an observer prior table without a gain table (builds with observer priors)
  exact    every other kernel (observer_gain_kernel, observe_kernel<true, true>, K1's shaped and nominal instantiations, ...),
           matched by its exact demangled name
and compared by instruction text (cuobjdump -sass without addresses and encodings).  Each differing line pair is classified:
  dfma-swap   one DFMA with its two factors exchanged (a*b+c = b*a+c)
  lds-swap    LDS.128 loads of unchanged addresses whose destination registers are permuted among themselves
  cbank       the same instruction reading a different offset of the parameter constant bank (c[0x0][...])
  other       anything else, including inserted or deleted instructions
The first two kinds also appear between two builds of the same sources.  A dfma-swap leaves the computed value unchanged; so does an
lds-swap whose loaded registers are only read as the two factors of the same products, which this script does not check: look at
the readers of the swapped registers (the listing of cuobjdump -sass) before calling one harmless."""
import collections
import difflib
import re
import subprocess
import sys

NAME = re.compile(r"^(?:void )?(ftocp_kernel|ftocp_sets_kernel)<(\d+), (\d+), 2, 4(?:, (true|false))?>")
DEFAULT = re.compile(r"^(?:void )?lmpc::(knn_ltv_regress_kernel|ss_select_kernel|shift_state_kernel|books_refresh_kernel|"
                     r"commit_laps_books_kernel|seed_books_kernel|pool_import_kernel|sim_step_kernel|commit_laps_kernel|"
                     r"seed_from_record_kernel|measure_kernel|pool_local_best_kernel|pool_export_kernel|nominal_model_kernel|observe_kernel)"
                     r"(<false>|<false, false>|<false, false, false>|<false, false, false, false>|<false, false, false, false, false>)?\(")
REPORTS = re.compile(r"^(?:void )?lmpc::(sim_step_kernel)<true(?:, false){1,2}>\(")
SURFACE = re.compile(r"^(?:void )?lmpc::(sim_step_kernel|nominal_model_kernel)<true>\(")
PRIOR = re.compile(r"^(?:void )?lmpc::(observe_kernel)<true(?:, false)?>\(")


def kernels(path):
    """{(variant, N, M): [instruction text]} of the QP kernels in a cubin or shared library"""
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in txt.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            k = NAME.match(name)
            d = DEFAULT.match(name)
            r = REPORTS.match(name)
            sf = SURFACE.match(name)
            pr = PRIOR.match(name)
            cur = None
            if k:
                sets = k.group(1) == "ftocp_sets_kernel" or k.group(4) == "true"
                cur = out.setdefault(("sets" if sets else "uniform", int(k.group(2)), int(k.group(3))), [])
            elif d:
                cur = out.setdefault(("default", d.group(1), 0), [])
            elif r:
                cur = out.setdefault(("reports", r.group(1), 0), [])
            elif sf:
                cur = out.setdefault(("surface", sf.group(1), 0), [])
            elif pr:
                cur = out.setdefault(("prior", pr.group(1), 0), [])
            else:
                cur = out.setdefault(("exact", name, 0), [])
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return out


def _ops(ins):
    op, _, rest = ins.partition(" ")
    return op, [o.strip() for o in rest.split(",")]


def compare(a, b):
    """Counter of the kinds of difference between two instruction lists (empty: identical)"""
    c = collections.Counter()
    lds = []   # (old, new) destination of each LDS.128 that loads the same address into another register
    cbank = re.compile(r"c\[0x0\]\[0x[0-9a-f]+\]")
    for tag, i1, i2, j1, j2 in difflib.SequenceMatcher(None, a, b, autojunk=False).get_opcodes():
        if tag == "equal":
            continue
        if tag != "replace" or i2 - i1 != j2 - j1:
            c["other"] += max(i2 - i1, j2 - j1)
            continue
        for x, y in zip(a[i1:i2], b[j1:j2]):
            ox, px = _ops(x)
            oy, py = _ops(y)
            if ox == oy == "LDS.128" and px[1:] == py[1:]:
                lds.append((px[0], py[0]))
            elif ox == oy and ox.startswith("DFMA") and len(px) == 4 and (px[0], px[3]) == (py[0], py[3]) and \
                    (px[1], px[2]) == (py[2], py[1]):
                c["dfma-swap"] += 1
            elif cbank.sub("c[0x0][]", x) == cbank.sub("c[0x0][]", y):
                c["cbank"] += 1
            else:
                c["other"] += 1
    if lds:
        c["lds-swap" if sorted(o for o, _ in lds) == sorted(n for _, n in lds) else "other"] += len(lds)
    return c


def main(old, new):
    ko, kn = kernels(old), kernels(new)
    totals = collections.defaultdict(collections.Counter)
    for key in sorted(set(ko) | set(kn)):
        variant, n, m = key
        label = ("%-24s" % n) if variant in ("default", "reports", "surface", "prior", "exact") else "<%2d,%2d>" % (n, m)
        if key not in ko or key not in kn:
            print("%-7s %s  only in %s" % (variant, label, "new" if key in kn else "old"))
            totals[variant]["unmatched"] += 1
            continue
        c = compare(ko[key], kn[key])
        verdict = "identical" if not c else ("other" if c["other"] else "+".join(sorted(c)))
        totals[variant][verdict] += 1
        print("%-7s %s  %5d instructions  %s%s" % (variant, label, len(kn[key]), verdict,
                                                  "" if not c else "  (" + ", ".join("%s %d" % kv for kv in sorted(c.items())) + " lines)"))
    for variant, t in sorted(totals.items()):
        print("%s: %d kernels: %s" % (variant, sum(t.values()), ", ".join("%d %s" % (v, k) for k, v in sorted(t.items()))))


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    main(sys.argv[1], sys.argv[2])
