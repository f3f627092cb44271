"""Builds libssd3d.so in-tree with nvcc for sm_90a (H100) (no torch / pybind dependency: the library is a plain
C-ABI shared object, see include/ssd3d.h)."""
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libssd3d.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-fmad=true",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.join(HERE, "..", "include", "ssd3d.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, defines=(), out=None):
    """defines / out: developer variants, e.g. build(True, defines=("TC_PROFILE", "SF_PROFILE", "SSD3D_DEV_HOOKS"),
    out="libssd3d_prof.so") -- loaded through the SSD3D_LIB environment variable by the probe tools; the product
    library is always built without defines."""
    if out is not None:
        return _build_to(os.path.join(HERE, out), os.path.join(HERE, "build_" + os.path.splitext(out)[0]), defines, verbose)
    if not force and not needs_build():
        return LIB
    return _build_to(LIB, os.path.join(HERE, "build"), (), verbose)


def _build_to(lib_path, obj_dir, defines, verbose):
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    os.makedirs(obj_dir, exist_ok=True)
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, out.decode()))
    cmd = [nvcc, "-shared", "-o", lib_path] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    return lib_path


if __name__ == "__main__":
    import sys
    if len(sys.argv) > 1 and sys.argv[1] == "dev":
        print(build(True, verbose=False, defines=("SSD3D_DEV_HOOKS",), out="libssd3d_dev.so"))
    elif len(sys.argv) > 1 and sys.argv[1] == "prof":
        print(build(True, verbose=True, defines=("TC_PROFILE", "SF_PROFILE", "SSD3D_DEV_HOOKS"), out="libssd3d_prof.so"))
    else:
        print(build(force=True, verbose=True))
