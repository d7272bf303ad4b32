"""Are the kernels at HEAD the same machine code as at <commit>?  (developer tool, no GPU needed)

Compiles csrc/<file>.cu of both trees for sm_90a and compares the SASS of every kernel the old tree defines,
instruction by instruction (addresses and encodings stripped).  Template parameters appended since then are matched
by trying the old mangled name with `Lb0E` (= false) inserted for each added bool.  Used at the end of round 1, after
the GPU budget was spent, to show that the host-side / opt-in changes made after the last GPU-verified commit left
every default kernel byte-identical.

    python tools/sass_identity.py 212bd74 embed_fm.cu gemm_tc.cu
"""
import hashlib
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr"]


def compile_tree(src_dir, inc_dir, name, out):
    subprocess.run(["nvcc", *FLAGS, "-I", inc_dir, "-I", src_dir, "-c", os.path.join(src_dir, name), "-o", out], check=True)


def kernels(obj):
    txt = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = hashlib.md5()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(.*?)\s*/\*", line)
        if m and cur:
            out[cur].update((" ".join(m.group(1).split()) + "\n").encode())
    return {k: v.hexdigest() for k, v in out.items()}


def main():
    commit, files = sys.argv[1], sys.argv[2:]
    tmp = tempfile.mkdtemp(prefix="sassid_")
    old_src = os.path.join(tmp, "old")
    os.makedirs(old_src)
    for f in os.listdir(os.path.join(ROOT, "deep_recommenders_b200", "csrc")):
        r = subprocess.run(["git", "-C", ROOT, "show", f"{commit}:deep_recommenders_b200/csrc/{f}"], capture_output=True)
        if r.returncode == 0:
            open(os.path.join(old_src, f), "wb").write(r.stdout)
    open(os.path.join(old_src, "deeprec_b200.h"), "wb").write(
        subprocess.run(["git", "-C", ROOT, "show", f"{commit}:include/deeprec_b200.h"], capture_output=True).stdout)
    total = diff = missing = 0
    for name in files:
        o_old, o_new = os.path.join(tmp, name + ".old.o"), os.path.join(tmp, name + ".new.o")
        compile_tree(old_src, old_src, name, o_old)
        compile_tree(os.path.join(ROOT, "deep_recommenders_b200", "csrc"), os.path.join(ROOT, "include"), name, o_new)
        ko, kn = kernels(o_old), kernels(o_new)
        for k, h in ko.items():
            cands = [k]
            for extra in (1, 2):      # bools appended to the template argument list since <commit> (all false by default)
                cands.append(re.sub(r"EEEv(?=[0-9N])", "E" + "Lb0E" * extra + "EEv", k, count=1))
            hit = next((c for c in cands if c in kn), None)
            total += 1
            if hit is None:
                missing += 1
                print("MISSING", name, k)
            elif kn[hit] != h:
                diff += 1
                print("DIFFERENT", name, k)
        print(f"{name}: {len(ko)} kernels at {commit}, {len(kn)} at HEAD")
    print(f"compared {total} kernels: {diff} differ, {missing} missing")
    sys.exit(1 if diff or missing else 0)


if __name__ == "__main__":
    main()
