"""What ptxas made of the wgmma chains of the fused kernels, per kernel, without a GPU.

    python tools/wgmma_report.py                      # every fused unit
    python tools/wgmma_report.py fused_sdf.cu         # some of them
    python tools/wgmma_report.py --all-kernels        # also the kernels that issue no wgmma

Each unit is compiled for sm_90a with the command and flags `build()` uses (`__graft_entry__.unit_cmd`, `UNITS`), plus
`-Xptxas -v`, into a temporary directory. Per kernel it prints the wgmma serialization diagnostics of ptxas (C7514: a non-wgmma
instruction reads accumulator registers inside a pipeline stage, C7515: one defines them, C7517: an injected wait, C7519: an injected
warpgroup.arrive, C7520: serialized by a compiler-inserted arrive in a divergent path), registers and spill bytes, and from
`cuobjdump -sass` the number of HGMMA instructions (the `HGMMA.64x8x16.F16 RZ` filler that closes a serialized group not counted)
and of `WARPGROUP.DEPBAR` waits. A chain that ptxas batched waits once per group; a serialized one waits after every HGMMA."""
import argparse
import os
import re
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

FUSED_UNITS = ("fused_sdf.cu", "fused_sdf_bwd.cu", "fused_rgb.cu", "fused_rgb_bwd.cu", "fused_bg.cu")
SERIALIZATION = ("C7514", "C7515", "C7517", "C7519", "C7520")
_TOOL = {t: shutil.which(t) or os.path.join("/usr/local/cuda/bin", t) for t in ("cuobjdump", "cu++filt")}


def _demangle(names):
    if not names:
        return {}
    r = subprocess.run([_TOOL["cu++filt"]], input="\n".join(names), stdout=subprocess.PIPE, text=True, check=True)
    out = r.stdout.splitlines()
    # without return type, namespaces and parameter list: k_sdf_fused_dual<3>
    short = []
    for d in out:
        d = re.sub(r"<unnamed>::|\(anonymous namespace\)::|\(int\)", "", d).replace("(bool)0", "false").replace("(bool)1", "true")
        short.append(re.sub(r"^void |\w+::", "", re.sub(r"\(.*$", "", d)))
    return dict(zip(names, short))


def parse_ptxas(log):
    """{mangled kernel: {"diag": {code: count}, "regs": int, "spill_st": int, "spill_ld": int}} from -Xptxas -v output"""
    k = {}

    def entry(name):
        return k.setdefault(name, {"diag": {}, "regs": None, "spill_st": None, "spill_ld": None})

    cur = None
    for line in log.splitlines():
        m = re.search(r"\((C75\d\d)\).*function '([^']+)'", line)
        if m:
            d = entry(m.group(2))["diag"]
            d[m.group(1)] = d.get(m.group(1), 0) + 1
            continue
        m = re.search(r"(?:Compiling entry function|Function properties for) '?([\w$]+)'?", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            e = entry(cur)
            e["spill_st"], e["spill_ld"] = int(m.group(1)), int(m.group(2))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            entry(cur)["regs"] = int(m.group(1))
    return k


def parse_sass(sass):
    """{mangled kernel: (HGMMA count without the RZ filler, WARPGROUP.DEPBAR count)} from cuobjdump -sass"""
    k, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            k[cur] = [0, 0]
            continue
        if cur is None:
            continue
        if re.search(r"\bHGMMA\.", line) and not re.search(r"HGMMA\.\S+ RZ,", line):
            k[cur][0] += 1
        elif "WARPGROUP.DEPBAR" in line:
            k[cur][1] += 1
    return {n: tuple(v) for n, v in k.items()}


def compile_unit(src, extra, outdir):
    obj = os.path.join(outdir, src.replace(".cu", ".o"))
    r = subprocess.run(graft.unit_cmd(src, obj, extra, verbose=True), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(src + " failed to compile:\n" + r.stdout)
    sass = subprocess.run([_TOOL["cuobjdump"], "-sass", obj], stdout=subprocess.PIPE, text=True, check=True).stdout
    return r.stdout, sass


def report(units=FUSED_UNITS):
    """[{"unit", "kernel", "mangled", "diag", "regs", "spill_st", "spill_ld", "hgmma", "depbar"}] of every kernel of `units`"""
    table = dict(graft.UNITS)
    missing = [u for u in units if u not in table]
    if missing:
        raise ValueError("not a unit of __graft_entry__.UNITS: " + ", ".join(missing))
    with tempfile.TemporaryDirectory(prefix="wgmma_report_") as tmp:
        with ThreadPoolExecutor(max_workers=max(1, min(len(units), os.cpu_count() or 1))) as ex:
            outs = list(ex.map(lambda u: compile_unit(u, table[u], tmp), units))
    rows = []
    for unit, (log, sass) in zip(units, outs):
        ptx, counts = parse_ptxas(log), parse_sass(sass)
        names = sorted(set(ptx) | set(counts))
        short = _demangle(names)
        for n in names:
            p = ptx.get(n, {"diag": {}, "regs": None, "spill_st": None, "spill_ld": None})
            h, d = counts.get(n, (0, 0))
            rows.append(dict(unit=unit, kernel=short[n], mangled=n, diag=p["diag"], regs=p["regs"], spill_st=p["spill_st"],
                             spill_ld=p["spill_ld"], hgmma=h, depbar=d))
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("units", nargs="*", default=list(FUSED_UNITS), help="translation units of __graft_entry__.UNITS")
    ap.add_argument("--all-kernels", action="store_true", help="also list kernels without HGMMA")
    args = ap.parse_args()
    rows = report(tuple(args.units))
    print(f"{'kernel':<44} {'unit':<18} {'regs':>4} {'spill st/ld':>11} {'HGMMA':>5} {'DEPBAR':>6}  diagnostics")
    for r in rows:
        if not (r["hgmma"] or args.all_kernels):
            continue
        diag = " ".join(f"{c}x{r['diag'][c]}" for c in SERIALIZATION if c in r["diag"]) or "-"
        spill = "-" if r["spill_st"] is None else f"{r['spill_st']}/{r['spill_ld']}"
        print(f"{r['kernel']:<44} {r['unit']:<18} {r['regs'] if r['regs'] is not None else '-':>4} {spill:>11} {r['hgmma']:>5} "
              f"{r['depbar']:>6}  {diag}")


if __name__ == "__main__":
    main()
