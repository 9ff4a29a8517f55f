"""The tests' native builds: g++ shared libraries of the shims that compile host / device headers on the CPU, and ptxas's resource report
of the product's kernels through nvcc with the product Makefile's flags (no GPU needed for either)."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess
import tempfile

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deepmimic_b200", "csrc")


def shared_library(src, flags):
    """ctypes.CDLL of the C++ file `src` built with `g++ <flags> -std=c++17 -shared -fPIC` into the temporary directory.  The library is
    named after a hash of the flags and of the source and every file it includes (as g++ -MM lists them), so it is rebuilt exactly when
    one of them changes; it is written under a temporary name and moved into place, so concurrent sessions never load a partial file."""
    cmd = ["g++"] + list(flags) + ["-std=c++17", "-x", "c++"]
    deps = subprocess.run(cmd + ["-MM", "-MT", "lib", src], stdout=subprocess.PIPE, check=True, text=True).stdout
    h = hashlib.sha1(" ".join(flags).encode())
    for f in deps.replace("\\\n", " ").split()[1:]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    name = os.path.splitext(os.path.basename(src))[0]
    so = os.path.join(tempfile.gettempdir(), "dm_%s_%d_%s.so" % (name, os.getuid(), h.hexdigest()[:16]))
    if not os.path.exists(so):
        tmp = "%s.%d.tmp" % (so, os.getpid())
        subprocess.check_call(cmd + ["-shared", "-fPIC", src, "-o", tmp])
        os.replace(tmp, so)
    return C.CDLL(so)


def nvcc():
    for p in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if p and os.path.isfile(p) and os.access(p, os.X_OK):
            return p
    return None


def makefile_flags():
    """NVFLAGS of the Makefile, $(ARCH) substituted"""
    mk = open(os.path.join(CSRC, "Makefile")).read()
    arch = re.search(r"^ARCH\s*:=\s*(.*)$", mk, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS\s*:=\s*(.*)$", mk, re.M).group(1).split()
    out = []
    for f in flags:
        out += arch if f == "$(ARCH)" else [f]
    return out


def ptxas_report(src, out_dir):
    """{entry: (registers, [(function, stack bytes, spill store bytes, spill load bytes), ...])}: the entry's register count, then the entry
    first and the routines ptxas lists with it"""
    r = subprocess.run([nvcc()] + makefile_flags() + ["-Xptxas", "-v", "-c", src, "-o", os.path.join(out_dir, "o.o")], cwd=CSRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    rep, entry = {}, None
    for m in re.finditer(r"Compiling entry function '(\S+)'|Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads|Used (\d+) registers", r.stdout):
        if m.group(1):
            entry = m.group(1)
            rep[entry] = (None, [])
        elif entry is None:
            continue
        elif m.group(6):
            rep[entry] = (int(m.group(6)), rep[entry][1])
        else:
            rep[entry][1].append((m.group(2), int(m.group(3)), int(m.group(4)), int(m.group(5))))
    return rep
