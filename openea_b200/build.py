"""In-tree build of liboea.so (sm_90a only) and of the CPU oracle.

`python -m openea_b200.build` or `__graft_entry__.build()`.  The .so files and object caches are build products
(git-ignored), rebuilt from the sources in the tree.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "_lib")
LIB_PATH = os.path.join(LIB_DIR, "liboea.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--compiler-options", "-fPIC",
    "-shared",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: liboea.so cannot be built")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    return h.hexdigest()


def _compile_one(job):
    src, obj, flags = job
    cmd = [_nvcc()] + flags + ["-c", "-o", obj, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    return src, res.returncode, res.stdout + res.stderr


def build_cuda(force=False, verbose=False, defines=(), out=None):
    """Compile every csrc/*.cu to an object (in parallel, cached per file on the digest of the file + all headers +
    flags) and link liboea.so.  `defines`/`out`: kernel A/B variants (scripts/ab_*.sh) built next to the default."""
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(LIB_DIR, exist_ok=True)
    out = out or LIB_PATH
    srcs = _sources()
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(ROOT, "include", "oea.h"))
    flags = [f for f in NVCC_FLAGS if f != "-shared"] + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else [])
    tag = hashlib.sha256(" ".join(flags).encode()).hexdigest()[:8]
    obj_dir = os.path.join(LIB_DIR, "obj_" + tag)
    os.makedirs(obj_dir, exist_ok=True)
    hdr_digest = _digest(hdrs)
    jobs, objs = [], []
    for src in srcs:
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        stamp = obj + ".sha256"
        digest = hashlib.sha256((hdr_digest + _digest([src])).encode()).hexdigest()
        objs.append(obj)
        fresh = os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read().strip() == digest
        if force or verbose or not fresh:
            jobs.append((src, obj, flags, stamp, digest))
    relink = bool(jobs) or not os.path.exists(out)
    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as pool:
            results = list(pool.map(_compile_one, [j[:3] for j in jobs]))
        failed = [r for r in results if r[1] != 0]
        for src, rc, text in results:
            if rc != 0 or verbose:
                sys.stderr.write(text)
        if failed:
            raise RuntimeError("nvcc failed building " + ", ".join(os.path.basename(r[0]) for r in failed))
        for _, obj, _, stamp, digest in jobs:
            with open(stamp, "w") as f:
                f.write(digest)
    if relink:
        cmd = [_nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out] + objs
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("nvcc failed linking liboea.so")
    return out


def build_oracle(force=False):
    """Compile the CPU oracle (test infrastructure, never used by the product path)."""
    odir = os.path.join(ROOT, "oracle")
    src = os.path.join(odir, "oea_oracle.c")
    out = os.path.join(odir, "liboea_oracle.so")
    if not os.path.exists(src):
        return None
    if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(src):
        return out
    cmd = ["gcc", "-O3", "-march=x86-64-v2", "-fopenmp", "-fPIC", "-shared", "-std=c11", "-o", out, src, "-lm"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("gcc failed building the oracle")
    return out


if __name__ == "__main__":
    print(build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_oracle(force="--force" in sys.argv))
