"""Compare the SASS of two versions of the CUDA library, kernel by kernel (no GPU needed).

    python scripts/sass_diff.py OLD NEW [NEW_NAME=OLD_NAME ...]

OLD and NEW are git revisions, or directories holding espnet_b200/csrc and include (the working tree: `.`).  Every .cu of each
version is compiled with the Makefile's flags plus `-Xptxas -v` and dumped with `cuobjdump -sass`.  Functions are matched by name,
with the per-file hash of the anonymous namespace stripped; NEW_NAME=OLD_NAME pairs rewrite parts of mangled NEW names, to match a
kernel whose template arguments changed with its old instance.  For every function of both versions the script reports whether its
instruction text and its ptxas registers, shared memory, stack and spills are identical, then lists the functions only one version
has.  It exits 1 if a common function differs or NEW has a function OLD lacks.
"""
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

# _ZN46_GLOBAL__N__122e3aba_13_search_ops_cu_7ee7b2de18beam_... : the namespace name and its length prefix carry per-build hashes
ANON = re.compile(r"\d+_(?:GLOBAL__N_|INTERNAL)_[0-9a-f]{8}_\d+_\w+?_cu_[0-9a-f]{8}")


def norm(name):
    return ANON.sub("<anon>", name)


def checkout(spec, dst):
    if os.path.isdir(spec):
        return os.path.abspath(spec)
    os.makedirs(dst)
    arch = subprocess.run(["git", "archive", spec, "espnet_b200/csrc", "include"], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", dst], input=arch, check=True)
    return dst


def makefile_flags(csrc):
    text = open(os.path.join(csrc, "Makefile")).read()
    var = dict(re.findall(r"^(\w+)\s*:?=\s*(.*)$", text, re.M))
    flags = var["NVFLAGS"].replace("$(ARCH)", var["ARCH"]).split()
    return flags, var["SRCS"].split()


def compile_one(csrc, flags, src, out):
    obj = os.path.join(out, src + ".o")
    p = subprocess.run(["nvcc", *flags, "-Xptxas", "-v", "-c", src, "-o", obj], cwd=csrc, capture_output=True, text=True, check=True)
    sass, res, cur = {}, {}, None
    for line in p.stderr.splitlines():   # ptxas -v: a "Function properties for F" line, then stack / spills, then registers / smem
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = norm(m.group(1))
            res[cur] = []
        elif cur and ("stack frame" in line or "Used" in line):
            res[cur].append(re.sub(r"^ptxas info\s*:\s*", "", line.strip()))
    dump = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    for fn in re.split(r"\n\s*Function : ", dump)[1:]:
        name, _, body = fn.partition("\n")
        # instruction + encoding lines; cuobjdump pads the columns to the widest line of the whole file, so whitespace is collapsed
        sass[norm(name.strip())] = [norm(" ".join(ln.split())) for ln in body.splitlines() if ln.strip().startswith("/*")]
    return sass, res


def compile_tree(root, out):
    csrc = os.path.join(root, "espnet_b200", "csrc")
    flags, srcs = makefile_flags(csrc)
    sass, res = {}, {}
    with ThreadPoolExecutor(os.cpu_count()) as pool:
        for s, r in pool.map(lambda src: compile_one(csrc, flags, src, out), srcs):
            sass.update(s)
            res.update(r)
    return sass, res


def main():
    old_spec, new_spec = sys.argv[1:3]
    renames = [a.split("=", 1) for a in sys.argv[3:]]
    with tempfile.TemporaryDirectory() as tmp:
        trees = [checkout(s, os.path.join(tmp, f"src{i}")) for i, s in enumerate((old_spec, new_spec))]
        outs = [os.path.join(tmp, f"obj{i}") for i in range(2)]
        for o in outs:
            os.makedirs(o)
        (old, old_res), (new, new_res) = (compile_tree(t, o) for t, o in zip(trees, outs))
    for a, b in renames:
        new = {k.replace(a, b): v for k, v in new.items()}
        new_res = {k.replace(a, b): v for k, v in new_res.items()}
    common = sorted(set(old) & set(new))
    bad = 0
    for name in common:
        same_sass, same_res = old[name] == new[name], old_res.get(name) == new_res.get(name)
        if not (same_sass and same_res):
            bad += 1
            print(f"DIFFERS  {name}: sass {'same' if same_sass else 'different'}, resources {old_res.get(name)} -> {new_res.get(name)}")
    print(f"common functions: {len(common)}, identical SASS and resources: {len(common) - bad}, differing: {bad}")
    for label, names in (("only in OLD", sorted(set(old) - set(new))), ("only in NEW", sorted(set(new) - set(old)))):
        print(f"{label}: {len(names)}")
        for n in names:
            print(f"  {n}  [{len(old.get(n) or new.get(n))} lines; {'; '.join((old_res if n in old else new_res).get(n, []))}]")
    sys.exit(1 if bad or set(new) - set(old) else 0)


if __name__ == "__main__":
    main()
