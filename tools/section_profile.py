"""Per-warp cycle breakdown of dm_step_kernel by code section (needs the profile build: `make -C deepmimic_b200/csrc profile`,
run with DM_LIB=deepmimic_b200/libdeepmimic_b200_prof.so).  Prints the average warp and the slowest warp of each block."""
import sys, os
import numpy as np
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch
from deepmimic_b200.assets import asset_root
from deepmimic_b200.capi import BatchedCore
N = 4096
root = asset_root(True)
core = BatchedCore(["--arg_file", "args/train_humanoid3d_spinkick_args.txt"], N, root, seed=1000)
A = core.dims.action_size
stream = torch.cuda.ExternalStream(core.stream())
with torch.cuda.stream(stream):
    off = torch.tensor(core.static(2), dtype=torch.float32, device="cuda"); scl = torch.tensor(core.static(3), dtype=torch.float32, device="cuda")
    lo = torch.tensor(core.static(4), dtype=torch.float32, device="cuda"); hi = torch.tensor(core.static(5), dtype=torch.float32, device="cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(7)
    core.set_episode_limit(20.0)
    core.reset(True, max_time=np.full(N, 20.0))
    for step in range(int(os.environ.get("PROF_PREROLL", "52"))):   # bench.py's preroll + warm-up: the steady-state mix of the 8(d) workload
        a = torch.clamp(-off + 0.25 / scl * torch.randn(N, A, device="cuda", generator=g), lo, hi).contiguous()
        core.set_action(a); core.update(1 / 600., 20); core.reset(False)
    a = torch.clamp(-off + 0.25 / scl * torch.randn(N, A, device="cuda", generator=g), lo, hi).contiguous()
    core.set_action(a); core.update(1 / 600., 20)
core.sync()
d = core.section_profile().astype(np.float64)   # [blocks, warps per block, 18] counters of the last launch
nblocks, warps_per_block = d.shape[:2]
print("%d blocks of %d warps" % (nblocks, warps_per_block))
# counter index -> section (dm_step_kernel's PROF / solve_rows' SPROF points).  7-9 are parts of solve_rows and already inside 10; 13-15 count rows.
names = {0: "kin", 1: "flags", 2: "sync (barriers)", 3: "clock/collide", 4: "PD solve+torque", 16: "sub-step 1 solve", 17: "sub-step 2 solve",
         5: "limit rows", 10: "solve_rows+z", 7: "  rows", 8: "  Abuild", 9: "  warm+PGS", 11: "dv_pass", 12: "integrate"}
timed = [0, 1, 2, 3, 4, 16, 17, 5, 10, 11, 12]
tot = d[:, :, timed].sum(axis=2)
print("cycles per launch (20 updates): mean warp %.0f, mean of slowest warp per block %.0f, max %.0f" % (tot.mean(), tot.max(axis=1).mean(), tot.max()))
wosync = tot - d[:, :, 2]
print("without barrier wait: mean warp %.0f, slowest per block %.0f" % (wosync.mean(), wosync.max(axis=1).mean()))
slow2 = d[np.arange(nblocks), wosync.argmax(axis=1)]
busy_tot = wosync.max(axis=1).mean()
print("%-22s %12s %12s %8s" % ("section", "mean warp", "busiest warp/block", "share"))
for k in timed[:8] + [7, 8, 9] + timed[8:]:
    print("%-22s %12.0f %12.0f %7.1f%%" % (names[k], d[:, :, k].mean(), slow2[:, k].mean(), 100.0 * slow2[:, k].mean() / busy_tot if k != 2 else 0.0))

nr_sum, nr_cnt = d[:, :, 13], d[:, :, 14]
busy = wosync.argmax(axis=1)
print("busiest warp per block: constraint sub-steps %.1f of 40, mean max-rows per such sub-step %.1f ; all warps: %.1f of 40, %.1f rows" % (
    nr_cnt[np.arange(nblocks), busy].mean(), (nr_sum[np.arange(nblocks), busy] / np.maximum(1, nr_cnt[np.arange(nblocks), busy])).mean(),
    nr_cnt.mean(), nr_sum.sum() / max(1, nr_cnt.sum())))
sr = d[:, :, 10]
print("solve_rows cycles per call: busiest %.0f, all %.0f" % ((sr[np.arange(nblocks), busy] / np.maximum(1, nr_cnt[np.arange(nblocks), busy])).mean(), sr.sum() / max(1, nr_cnt.sum())))

# ---- where does the single wave end?  kernel time = the slowest block; a block's time = sum over stages of its slowest warp (barrier after every stage)
bt = tot.max(axis=1)
print("block time (max warp incl. barrier wait) percentiles: p10 %.0f p50 %.0f p90 %.0f p99 %.0f max %.0f ; mean/max = %.2f" % (
    np.percentile(bt, 10), np.percentile(bt, 50), np.percentile(bt, 90), np.percentile(bt, 99), bt.max(), bt.mean() / bt.max()))
gen = d[:, :, 15]
print("general-path (> W rows) solve calls per launch: total %d, per block mean %.2f max %d" % (gen.sum(), gen.sum(axis=1).mean(), gen.sum(axis=1).max()))
order = np.argsort(-bt)
print("slowest blocks: block, time, busiest-warp work (no wait), its constraint sub-steps, its mean rows, general-path calls in block, sum of all warps' work")
for b in list(order[:6]) + list(order[len(order) // 2: len(order) // 2 + 3]):
    w = wosync[b].argmax()
    print("  block %3d time %9.0f busiest work %9.0f substeps %2d rows %.1f general %2d block work %10.0f | busiest warp sections: %s" % (
        b, bt[b], wosync[b, w], nr_cnt[b, w], nr_sum[b, w] / max(1, nr_cnt[b, w]), gen[b].sum(), wosync[b].sum(),
        " ".join("%s=%.0f" % (names[k].strip().replace(" ", "_"), d[b, w, k]) for k in (0, 3, 4, 16, 17, 7, 8, 9, 10, 11, 12))))
c = np.corrcoef(bt, gen.sum(axis=1))[0, 1] if gen.sum() > 0 else 0.0
c2 = np.corrcoef(bt, nr_sum.sum(axis=1))[0, 1]
c3 = np.corrcoef(bt, wosync.max(axis=1))[0, 1]
print("correlation of block time with: general-path calls %.2f, total rows in block %.2f, busiest warp's own work %.2f" % (c, c2, c3))
