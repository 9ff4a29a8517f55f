"""Resources of the step kernel as ptxas reports them (no GPU needed): the imitate instantiations keep nothing of their main loop in local
memory around the phase calls.  The routines take nearly all 128 registers and ptxas fits the caller's live values around them; once those
values no longer fit, every stage stored and reloaded them through the stack.  Their only stack is the scratch array of the double-precision
sin / cos argument reduction (kin_wrap_sync, clip wraps), which a one-line probe kernel measures with the same flags."""
import os
import re

import pytest

from tests.native import nvcc, ptxas_report


@pytest.mark.skipif(nvcc() is None, reason="needs nvcc")
@pytest.mark.parametrize("w", [16, 32])
def test_imitate_step_kernel_keeps_its_loop_out_of_local_memory(w, tmp_path):
    probe = tmp_path / "probe.cu"
    probe.write_text("__global__ void probe(double* p) { p[0] = sin(p[0]) + cos(p[1]); }\n")
    scratch = ptxas_report(str(probe), str(tmp_path))
    (trig_frame,) = [f[1] for _, fs in scratch.values() for f in fs if f[0] == "_Z5probePd"]
    rep = ptxas_report(os.path.join("kernels", "dm_step.cu"), str(tmp_path))
    (entry,) = [e for e in rep if re.search(r"dm_step_kernelILi%dELb0E" % w, e)]
    funcs = rep[entry][1]
    assert funcs[0][0] == entry and len(funcs) > 5, funcs
    assert funcs[0][1] == trig_frame, "stack frame %d B, the sin / cos scratch alone is %d B" % (funcs[0][1], trig_frame)
    for name, _, stores, loads in funcs:
        assert stores == 0 and loads == 0, "%s: %d B spill stores, %d B spill loads" % (name, stores, loads)
