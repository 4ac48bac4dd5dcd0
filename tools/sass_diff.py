"""Per-kernel SASS comparison of the working tree against a git revision (default HEAD): both trees' rend3_b200/csrc are compiled
with build()'s nvcc flags (__graft_entry__.py) into temporary directories, every kernel's `cuobjdump -sass` is normalised (addresses,
encodings and the per-file hashes of anonymous-namespace names stripped) and the kernels are compared one by one.  For a kernel that
differs it prints the resource usage on both sides (registers, stack, local memory: spills show there) and whether the floating-point
instructions are the same multiset and in the same order.  A refactor that should leave the machine code alone is checked with it.

    python tools/sass_diff.py [REV] [--show]      (--show prints a unified diff of every kernel that differs)
"""
import concurrent.futures
import difflib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as entry  # noqa: E402

CUOBJDUMP = os.path.join(os.path.dirname(entry.NVCC), "cuobjdump")


def export(rev, dst):
    """rend3_b200/csrc and include/ of `rev` under dst (a relative include path in the sources points at ../../include)."""
    archive = subprocess.run(["git", "-C", ROOT, "archive", rev, "rend3_b200/csrc", "include"], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", dst], input=archive, check=True)
    return os.path.join(dst, "rend3_b200", "csrc")


def compile_tree(csrc, out):
    def one(item):
        src, extra = item
        o = os.path.join(out, os.path.splitext(src)[0] + ".o")
        r = subprocess.run([entry.NVCC, "-x", "cu", "-c", os.path.join(csrc, src), "-o", o] + entry.COMMON + extra, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {csrc}/{src}:\n{r.stderr}")
        return src, o
    with concurrent.futures.ThreadPoolExecutor(os.cpu_count() or 4) as pool:
        # a source the other tree does not have yet (a new unit) is compiled on one side only: its kernels show as ONLY IN
        return dict(pool.map(one, [s for s in entry.SOURCES if os.path.exists(os.path.join(csrc, s[0]))]))


def unhash(text):
    """Names in anonymous namespaces carry hashes of the compiled file's path (<len>_GLOBAL__N__<hash>_<n>_<file>_<suffix>, and the same
    with _INTERNAL_): keep the file name only.  <len> is the length of the whole identifier, <n> that of <file>."""
    out, pos = [], 0
    for m in re.finditer(r"(\d+)(_GLOBAL__N__|_INTERNAL_)[0-9a-f]{8}_(\d+)_", text):
        if m.start() < pos:
            continue
        name = text[m.end():m.end() + int(m.group(3))]
        out += [text[pos:m.start()], m.group(2), name]
        pos = m.start(2) + int(m.group(1))
    return "".join(out) + text[pos:]


def kernels(obj):
    """{normalised kernel name: (mangled name, [normalised instructions])} of one object file."""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    fns, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = unhash(m.group(1))
            fns[cur] = (m.group(1), [])
        elif cur and "/*" in line and ";" in line:
            fns[cur][1].append(unhash(line.split("*/", 1)[1].split(";")[0].strip()))
    return fns


def resources(obj):
    """{normalised kernel name: "REG:.. STACK:.. LOCAL:.."} of one object file (cuobjdump -res-usage)."""
    out = subprocess.run([CUOBJDUMP, "-res-usage", obj], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = unhash(m.group(1))
        elif cur and "REG:" in line:
            res[cur] = " ".join(f for f in line.split() if f.split(":")[0] in ("REG", "STACK", "SHARED", "LOCAL"))
            cur = None
    return res


def fp_ops(instructions):
    """The floating-point instructions' opcodes with their modifiers (rounding, comparison), in program order: a change of schedule or
    register allocation keeps the multiset, a change of arithmetic does not."""
    ops = [re.sub(r"^@!?U?P\w+\s+", "", i).split()[0] for i in instructions]
    return [o for o in ops if re.match(r"(F[A-Z]+|MUFU|HADD2|HMUL2|HFMA2(?!\.MMA)|DADD|DMUL|DFMA)\b", o)]


def strip_targets(instructions):
    """Branch targets are offsets into the kernel: one inserted instruction moves all later ones, which --show should not list."""
    return [re.sub(r"0x[0-9a-f]+", "0x?", i) if re.match(r"(@!?U?P\w+\s+)?(BRA|BSSY|CALL|BRX|JMP)\b", i) else i for i in instructions]


def demangle(name):
    return subprocess.run(["cu++filt", name], capture_output=True, text=True).stdout.strip() or name


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    show = "--show" in sys.argv
    rev = args[0] if args else "HEAD"
    with tempfile.TemporaryDirectory() as tmp:
        dirs = {k: os.path.join(tmp, k) for k in ("base_src", "base_obj", "tree_obj")}
        for d in dirs.values():
            os.makedirs(d)
        base = compile_tree(export(rev, dirs["base_src"]), dirs["base_obj"])
        tree = compile_tree(os.path.join(ROOT, "rend3_b200", "csrc"), dirs["tree_obj"])
        same = differ = 0
        for src, _ in entry.SOURCES:
            a, b = (kernels(base[src]) if src in base else {}), kernels(tree[src])
            ra, rb = (resources(base[src]) if src in base else {}), resources(tree[src])
            for name in sorted(set(a) | set(b)):
                label = f"{src}: {demangle((a.get(name) or b.get(name))[0])[:140]}"
                if name not in a or name not in b:
                    print(f"ONLY IN {'tree' if name in b else rev}  {label}")
                    differ += 1
                    continue
                old, new = a[name][1], b[name][1]
                if old == new:
                    same += 1
                else:
                    differ += 1
                    fa, fb = fp_ops(old), fp_ops(new)
                    print(f"DIFFERS  {label}\n         {len(old)} -> {len(new)} instructions; {ra.get(name)} -> {rb.get(name)}; "
                          f"floating-point instructions {len(fa)} -> {len(fb)}, same multiset: {sorted(fa) == sorted(fb)}, same order: {fa == fb}")
                    if show:
                        diff = difflib.unified_diff(strip_targets(old), strip_targets(new), rev, "tree", n=2, lineterm="")
                        sys.stdout.writelines(l + "\n" for l in diff)
        print(f"{same} kernels identical, {differ} differ ({rev} vs working tree)")


if __name__ == "__main__":
    main()
