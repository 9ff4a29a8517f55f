"""Device-clock time of the tensor-core learner's step split for data-parallel training (TensorCoreLearner.grad + apply) against the fused
step, for the plain actor (227 inputs, 28 actions), the critic (227 inputs) and the AMP discriminator (226 inputs), 1024-512 hidden units (the
spin-kick and imitate_amp humanoid3d sizes), at minibatch 1024 and 4096 (the discriminator: that many agent and as many expert rows), on
random weights and inputs; and one torch.distributed all-reduce of each network's flat gradient.  Prints the card and its power limit.

Under torchrun (one process per GPU) the all-reduce runs over all ranks on NCCL; run alone, the group has one rank, so the all-reduce time
is NCCL's single-rank cost, not a multi-GPU figure.

    python tools/data_parallel_time.py [--repeat 50]
    torchrun --nproc_per_node 8 tools/data_parallel_time.py"""
import argparse
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import torch
    import torch.distributed as dist
    from deepmimic_b200.capi import DmLearnBatch, DmLearnDiscBatch, TensorCoreLearner
    from deepmimic_b200.rollout import build_critic, build_discriminator, build_policy
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("data_parallel_time.py needs a CUDA device")
    rank = int(os.environ.get("RANK", 0))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
    if "WORLD_SIZE" in os.environ:
        dist.init_process_group("nccl")
    else:
        dist.init_process_group("nccl", init_method="file://" + os.path.join(tempfile.mkdtemp(), "init"), rank=0, world_size=1)
    world = dist.get_world_size()
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        print("device: %s; nvidia-smi: %s; all-reduce world %d" % (torch.cuda.get_device_name(), q.stdout.strip() or "n/a", world))
    S, A, M, R = 227, 28, 226, 32 * 4096
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    g = torch.Generator(device=dev).manual_seed(1)
    rnd = lambda *shape: torch.randn(*shape, device=dev, generator=g)
    states, norm_a, amp = rnd(R, S), 0.3 * rnd(R, A), rnd(R, M)
    old_logp, adv, tar = rnd(R) - 20.0, rnd(R), rnd(R)
    zeros, ones = torch.zeros(S, device=dev), torch.ones(S, device=dev)
    logstd = torch.full((A,), -1.6, device=dev)
    lo, hi = torch.full((A,), -2.0, device=dev), torch.full((A,), 2.0, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n):
        for _ in range(3):
            fn()
        torch.cuda.synchronize(); e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    p = lambda x: x.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    for kind, net in (("actor", build_policy(S, A)), ("critic", build_critic(S)), ("disc", build_discriminator(M))):
        net = net.to(dev)
        for B in (1024, 4096):
            acc = {q: torch.zeros_like(q) for q in net.parameters()}
            tc = TensorCoreLearner(net, acc, kind, 2 * B if kind == "disc" else B, device=dev.index)
            tc.set_weights(stream=st)
            idx = torch.randint(0, R, (B,), device=dev, generator=g)
            stats = torch.zeros(6, device=dev)
            if kind == "disc":
                batch = DmLearnDiscBatch(agent=p(amp), expert=p(amp), agent_idx=p(idx), expert_idx=p(idx.flip(0).contiguous()), rows=B,
                                         in_mean=p(zeros), in_istd=p(ones), in_clip=0.0, stepsize=1e-6, momentum=0.9, weight_decay=1e-4,
                                         logit_reg_weight=0.05, grad_penalty_weight=5.0, stats=p(stats))
            else:
                batch = DmLearnBatch(states=p(states), idx=p(idx), rows=B, in_mean=p(zeros), in_istd=p(ones), in_clip=0.0, norm_actions=p(norm_a),
                                     old_logp=p(old_logp), adv=p(adv), logstd=p(logstd), bound_min=p(lo), bound_max=p(hi), ratio_clip=0.2,
                                     norm_targets=p(tar), stepsize=1e-7, momentum=0.9, weight_decay=5e-4, stats=p(stats))
            flat = torch.empty(tc.grad_size(), device=dev)
            t_fused = timed(lambda: tc.step(batch, stream=st), a.repeat)
            t_grad = timed(lambda: tc.grad(batch, flat, stream=st), a.repeat)
            t_apply = timed(lambda: tc.apply(batch, flat, 1.0, stream=st), a.repeat)
            t_split = timed(lambda: (tc.grad(batch, flat, stream=st), tc.apply(batch, flat, 1.0, stream=st)), a.repeat)
            t_ar = timed(lambda: dist.all_reduce(flat), a.repeat)
            if rank == 0:
                print("%-6s minibatch %4d: fused step %7.3f ms; grad %7.3f + apply %6.3f ms, grad + apply %7.3f ms (%+.1f%%); "
                      "all-reduce of %d floats (%.2f MB) %7.3f ms"
                      % (kind, B, t_fused, t_grad, t_apply, t_split, 100.0 * (t_split / t_fused - 1.0), flat.numel(), flat.numel() * 4 / 2 ** 20, t_ar))
            tc.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
