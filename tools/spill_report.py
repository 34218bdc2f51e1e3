"""Register / spill report of the mapper kernels, from the compiler alone (no GPU needed).

Compiles uncalled_b200/csrc/unc_abi.cu for sm_90a with the library's own nvcc flags plus -Xptxas -v, then prints for
k2_map, k2_map_ord, k2_map_stream and the exact-ties kernels k2_map_exact and k2_map_stream_exact:
  * registers, stack frame and spill bytes as ptxas reports them;
  * the local-memory instructions (LDL / STL) of the kernel's SASS per source line, from `nvdisasm -g` on the cubin
    (inlined code is attributed to the line of the inlined function, which is where the spill sits).

    python tools/spill_report.py                 # compile and report
    python tools/spill_report.py -D K2_WARPS=16  # the same for another CTA shape
"""
import argparse, collections, os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "uncalled_b200", "csrc", "unc_abi.cu")
KERNELS = ("k2_map", "k2_map_ord", "k2_map_stream", "k2_map_exact", "k2_map_stream_exact")


def nvcc_flags():
    sys.path.insert(0, ROOT)
    from uncalled_b200._native import NVCC_FLAGS
    f = list(NVCC_FLAGS)                               # a cubin of the one translation unit: no host / link flags
    i = f.index("-Xcompiler")
    del f[i:i + 2]
    f.remove("--shared")
    return f


def compile_cubin(out_dir, defines=()):
    """-> (cubin path, ptxas -v text)"""
    cubin = os.path.join(out_dir, "unc_abi.cubin")
    cmd = ["nvcc", "-cubin", "-Xptxas", "-v"] + nvcc_flags() + ["-D" + d for d in defines] + ["-o", cubin, SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return cubin, r.stdout + r.stderr


def demangled_name(mangled):
    m = re.match(r"_Z(\d+)", mangled)
    return mangled[len(m.group(0)):len(m.group(0)) + int(m.group(1))] if m else mangled


def ptxas_stats(text):
    """{kernel: {"regs", "stack", "spill_st", "spill_ld"}} from `ptxas -v` output"""
    res, cur, props = {}, None, None
    for l in text.split("\n"):
        m = re.search(r"Compiling entry function '(\S+)'", l)
        if m:
            cur = demangled_name(m.group(1))
            res[cur] = {}
            continue
        if cur is None:
            continue
        m = re.search(r"Function properties for (\S+)", l)
        if m:                                          # the kernel's own, or those of a non-inlined callee (unc_pdq_sort)
            props = demangled_name(m.group(1))
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", l)
        if m and props == cur:
            res[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", l)
        if m:
            res[cur]["regs"] = int(m.group(1))
    return res


def spill_lines(cubin, kernels=KERNELS):
    """{kernel: Counter{(file, line): [n_ldl, n_stl]}} from `nvdisasm -g`"""
    out = subprocess.run(["nvdisasm", "-g", "-c", cubin], capture_output=True, text=True, check=True).stdout
    res, kern, loc = {}, None, ("?", 0)
    for l in out.split("\n"):
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", l)
        if m:
            name = demangled_name(m.group(1))
            kern = name if name in kernels else None
            if kern:
                res[kern] = collections.defaultdict(lambda: [0, 0])
            continue
        if kern is None:
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', l)
        if m:
            loc = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?(LDL|STL)\b", l)
        if m:
            res[kern][loc][0 if m.group(1) == "LDL" else 1] += 1
    return res


def report(stats, lines, kernels=KERNELS):
    print("%-20s %5s %6s %9s %9s %6s %6s" % ("kernel", "regs", "stack", "spill_st", "spill_ld", "LDL", "STL"))
    for k in kernels:
        s, ln = stats.get(k, {}), lines.get(k, {})
        print("%-20s %5s %6s %9s %9s %6d %6d" % (k, s.get("regs"), s.get("stack"), s.get("spill_st"), s.get("spill_ld"),
                                                 sum(v[0] for v in ln.values()), sum(v[1] for v in ln.values())))
    for k in kernels:
        ln = lines.get(k, {})
        if not ln:
            continue
        print("\n## %s: LDL / STL per source line" % k)
        for (f, n), (ld, st) in sorted(ln.items()):
            print("   %-22s %5d   LDL %3d  STL %3d" % (f, n, ld, st))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("-D", dest="defines", action="append", default=[], help="extra preprocessor definition (NAME=VAL)")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        cubin, text = compile_cubin(d, a.defines)
        report(ptxas_stats(text), spill_lines(cubin))


if __name__ == "__main__":
    main()
