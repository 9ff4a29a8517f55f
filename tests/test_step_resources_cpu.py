"""Resources of the step kernel as ptxas reports them (no GPU needed): the imitate instantiations keep nothing of their main loop in local
memory around the phase calls.  The routines take nearly all 128 registers and ptxas fits the caller's live values around them; once those
values no longer fit, every stage stored and reloaded them through the stack.  Their only stack is the scratch array of the double-precision
sin / cos argument reduction (kin_wrap_sync, clip wraps), which a one-line probe kernel measures with the same flags."""
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "deepmimic_b200", "csrc")


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
    """{entry: [(function, stack bytes, spill store bytes, spill load bytes), ...]}: the entry first, then the routines ptxas lists with it"""
    r = subprocess.run([nvcc()] + makefile_flags() + ["-Xptxas", "-v", "-c", src, "-o", os.path.join(out_dir, "o.o")], cwd=CSRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    rep, entry = {}, None
    for m in re.finditer(r"Compiling entry function '(\S+)'|Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                         r.stdout):
        if m.group(1):
            entry = m.group(1)
            rep[entry] = []
        elif entry is not None:
            rep[entry].append((m.group(2), int(m.group(3)), int(m.group(4)), int(m.group(5))))
    return rep


@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
@pytest.mark.parametrize("w", [16, 32])
def test_imitate_step_kernel_keeps_its_loop_out_of_local_memory(w, tmp_path):
    probe = tmp_path / "probe.cu"
    probe.write_text("__global__ void probe(double* p) { p[0] = sin(p[0]) + cos(p[1]); }\n")
    scratch = ptxas_report(str(probe), str(tmp_path))
    (trig_frame,) = [f[1] for fs in scratch.values() for f in fs if f[0] == "_Z5probePd"]
    rep = ptxas_report(os.path.join("kernels", "dm_step.cu"), str(tmp_path))
    (entry,) = [e for e in rep if re.search(r"dm_step_kernelILi%dELb0E" % w, e)]
    funcs = rep[entry]
    assert funcs[0][0] == entry and len(funcs) > 5, funcs
    assert funcs[0][1] == trig_frame, "stack frame %d B, the sin / cos scratch alone is %d B" % (funcs[0][1], trig_frame)
    for name, _, stores, loads in funcs:
        assert stores == 0 and loads == 0, "%s: %d B spill stores, %d B spill loads" % (name, stores, loads)
