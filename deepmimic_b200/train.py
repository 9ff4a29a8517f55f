"""Train a skill: the counterpart of the reference's `DeepMimic_Optimizer.py --arg_file args/train_*_args.txt` (one GPU) and of its
`mpi_run.py --num_workers N` (one process per GPU under torchrun).

    python -m deepmimic_b200.train --arg_file args/train_humanoid3d_spinkick_args.txt [reference arguments ...]
        [--asset_root DIR] [--num_envs 4096] [--window_steps 32] [--max_iters K] [--backend tensor_core] [--seed 0] [--device 0] [--resume PATH]
    torchrun --nproc-per-node 8 -m deepmimic_b200.train ... --num_envs 32768

Under torchrun (WORLD_SIZE > 1) every rank joins an NCCL group on the GPU of its LOCAL_RANK (--device is ignored) and the Trainer splits
--num_envs, the job's total, between the ranks (deepmimic_b200/trainer.py: Trainer, process_group).  Only the first rank prints and writes the
log; rank r > 0 writes its checkpoints next to the first rank's, with .rank<r> before the .pt, and --resume PATH (the first rank's file)
reads each rank's own.

Every argument this module does not name goes to the scene, as the reference's arguments do.  --agent_files, --output_path and
--int_output_path are read from the same argument list, the command line before the arg file (the reference's ArgParser keeps the first value
of a key), and so is --model_files: a reference TensorBundle prefix or a Trainer checkpoint whose networks and normalisers the run starts from
(deepmimic_b200/model_files.py), at iteration 0.  Such a run resumes with the arguments it started with, --model_files included: the
checkpoint records the model files, and --resume refuses a checkpoint of a run that started from other ones (or from none).  The log goes to <output_path>/agent0_log.txt and the checkpoint to <output_path>/agent0_checkpoint.pt (every OutputIters iterations
and at the end); with --int_output_path, an intermediate checkpoint every IntOutputIters iterations goes to
<int_output_path>/agent0_int_checkpoint_<iteration>.pt.  --resume continues a checkpoint of the same run (arguments, agent file, num_envs,
window_steps, backend, seed), its log and its iteration numbering.

Training under pushes: --push_force LO,HI (N), --push_bodies B1[,B2...] (body ids), --push_duration LO,HI (s) and --push_interval LO,HI (s, the
gap after the previous push), all four or none, push every training environment at random (DeepMimicBatchEnv.set_push_schedule): after each
push its environment waits a gap drawn from the interval, then a body from the list is pushed horizontally with a magnitude and for a duration
drawn from their ranges.  The evaluation (Test_Return) runs without pushes.  The schedule is part of the run record: --resume needs the same
four options.

Training under randomised dynamics: --rand_friction, --rand_kp, --rand_kd, --rand_torque_limit and --rand_mass LO,HI, each optional (any one
switches randomisation on, a kind not given stays 1), draw every training environment's factors at every reset
(DeepMimicBatchEnv.set_dynamics_randomization; --rand_mass draws one factor per body).  The evaluation (Test_Return) runs on the nominal
model.  The bounds are part of the run record: --resume needs the same options.  They combine with the push options.

Training under control latency: --rand_latency LO,HI (s) draws every training environment's actuation delay at every reset, a whole number of
1/600 s updates between LO and HI rounded to the nearest update, at most 19 updates (0.0317 s) (DeepMimicBatchEnv.set_action_latency_randomization).
The evaluation (Test_Return) runs without delay.  The bounds are part of the run record: --resume needs the same option.  It combines with the
push and dynamics options.
"""
import argparse
import math
import os
import re
import sys


def parse_arg_list(tokens):
    """the reference's ArgParser over a token list: --key followed by its values; '#'-prefixed tokens are comments; the first occurrence of a
    key wins"""
    table, key, vals = {}, None, []
    for tok in tokens:
        if tok.startswith("#"):
            continue
        if tok.startswith("--"):
            if key is not None and key not in table:
                table[key] = vals
            key, vals = tok[2:], []
        else:
            vals.append(tok)
    if key is not None and key not in table:
        table[key] = vals
    return table


def _file_tokens(path):
    """the tokens of an arg file: lines starting with '#' are comments"""
    out = []
    with open(path) as f:
        for line in re.split(r"[\n\r]+", f.read()):
            if line and not line.lstrip().startswith("#"):
                out += line.split()
    return out


def _resolve(asset_root, path):
    """a path of the argument list: absolute, under the asset root, or relative to the working directory.  A TensorBundle prefix (a model
    file) counts as existing when its .index file does."""
    if os.path.isabs(path):
        return path
    under = os.path.join(asset_root, path)
    return under if os.path.exists(under) or os.path.exists(under + ".index") else path


def arg_table(scene_args, asset_root, prog="train"):
    """{key: values} of the scene arguments and the arg file they name, the command line first (parse_arg_list's rule)"""
    table = parse_arg_list(scene_args)
    if "arg_file" in table and table["arg_file"]:
        arg_file = _resolve(asset_root, table["arg_file"][0])
        if not os.path.exists(arg_file):
            raise SystemExit("%s: arg file %s not found" % (prog, table["arg_file"][0]))
        for k, v in parse_arg_list(_file_tokens(arg_file)).items():
            table.setdefault(k, v)
    return table


def first_arg(table, key):
    """the first value of `key` in an arg_table, "" without one"""
    return table[key][0] if table.get(key) else ""


def resolve_args(scene_args, asset_root):
    """(agent file, output path, int output path) from the scene arguments and the arg file they name (command line first)"""
    table = arg_table(scene_args, asset_root)
    if not first_arg(table, "agent_files"):
        raise SystemExit("train: no --agent_files in the arguments or the arg file")
    return _resolve(asset_root, first_arg(table, "agent_files")), first_arg(table, "output_path") or "output", first_arg(table, "int_output_path")


def resolve_model_files(scene_args, asset_root, prog="train"):
    """--model_files of the scene arguments or their arg file (command line first), resolved like the other paths; None without one"""
    m = first_arg(arg_table(scene_args, asset_root, prog), "model_files")
    return _resolve(asset_root, m) if m else None


def parse_range(text):
    """LO,HI: two finite numbers >= 0 with LO <= HI"""
    try:
        v = [float(x) for x in text.split(",")]
    except ValueError:
        v = []
    if len(v) != 2 or not all(math.isfinite(x) and x >= 0.0 for x in v) or v[0] > v[1]:
        raise argparse.ArgumentTypeError("need LO,HI: two finite numbers >= 0 with LO <= HI, got %r" % text)
    return v


def parse_bodies(text):
    """B1[,B2...]: 1 to 32 body ids >= 0"""
    try:
        v = [int(x) for x in text.split(",")]
    except ValueError:
        v = []
    if not 1 <= len(v) <= 32 or min(v) < 0:
        raise argparse.ArgumentTypeError("need 1 to 32 comma-separated body ids >= 0, got %r" % text)
    return v


PUSH_OPTIONS = ("push_force", "push_bodies", "push_duration", "push_interval")


def push_schedule(opts):
    """the Trainer's push_schedule from the four push options: None without them; all four or none"""
    given = [k for k in PUSH_OPTIONS if getattr(opts, k) is not None]
    if not given:
        return None
    if len(given) != len(PUSH_OPTIONS):
        raise SystemExit("train: --%s need each other: missing %s" % (", --".join(PUSH_OPTIONS),
                                                                     ", ".join("--" + k for k in PUSH_OPTIONS if k not in given)))
    return dict(bodies=opts.push_bodies, force=opts.push_force, duration=opts.push_duration, gap=opts.push_interval)


RAND_OPTIONS = ("rand_friction", "rand_kp", "rand_kd", "rand_torque_limit", "rand_mass")


def dynamics_randomization(opts):
    """the Trainer's dynamics_randomization from the --rand_* options: None without any; a kind not given stays (1, 1)"""
    given = {k[len("rand_"):]: getattr(opts, k) for k in RAND_OPTIONS if getattr(opts, k) is not None}
    if given.get("mass") is not None and not given["mass"][0] > 0.0:
        raise SystemExit("train: --rand_mass needs LO > 0, got %g" % given["mass"][0])
    return given or None


def parse_latency_range(text):
    """LO,HI seconds: each rounds to a whole update in [0, 19] (0 to 0.0317 s), LO <= HI"""
    from .capi import UPDATES_PER_ACTION, latency_updates
    v = parse_range(text)
    try:
        for x in v:
            latency_updates(x, UPDATES_PER_ACTION)
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e))
    return v


def build_parser():
    ap = argparse.ArgumentParser(prog="python -m deepmimic_b200.train", description=__doc__.split("\n\n")[0], allow_abbrev=False)
    ap.add_argument("--asset_root", default=None, help="the reference's data / args tree (default: the bundled asset archive)")
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--window_steps", type=int, default=32, help="policy steps per environment in each iteration's window")
    ap.add_argument("--max_iters", type=int, default=None, help="stop after this many iterations in all (default: run until interrupted)")
    ap.add_argument("--backend", default="tensor_core", choices=("tensor_core", "torch"))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--resume", default=None, help="a checkpoint of the same run to continue")
    ap.add_argument("--push_force", type=parse_range, default=None, metavar="LO,HI", help="training under pushes: push magnitude range in N")
    ap.add_argument("--push_bodies", type=parse_bodies, default=None, metavar="B1[,B2...]", help="training under pushes: the bodies pushed")
    ap.add_argument("--push_duration", type=parse_range, default=None, metavar="LO,HI", help="training under pushes: push length range in s")
    ap.add_argument("--push_interval", type=parse_range, default=None, metavar="LO,HI",
                    help="training under pushes: range of the gap after an environment's previous push in s")
    for k, what in (("friction", "contact friction"), ("kp", "every PD controller's Kp"), ("kd", "every PD controller's Kd"),
                    ("torque_limit", "every joint's torque limit"), ("mass", "every body's mass (one factor per body)")):
        ap.add_argument("--rand_" + k, type=parse_range, default=None, metavar="LO,HI",
                        help="training under randomised dynamics: range of the factor on %s, drawn per environment at every reset" % what)
    ap.add_argument("--rand_latency", type=parse_latency_range, default=None, metavar="LO,HI",
                    help="training under control latency: range of the actuation delay in s (whole 1/600 s updates, at most 0.0317 s), drawn per "
                         "environment at every reset")
    return ap


def rank_path(path, rank):
    """the checkpoint file of `rank` for the first rank's `path`: path itself for rank 0, <stem>.rank<r>.pt otherwise"""
    if rank == 0:
        return path
    stem, ext = os.path.splitext(path)
    return "%s.rank%d%s" % (stem, rank, ext or ".pt")


def main(argv=None):
    from .assets import asset_root as default_asset_root
    from .sharding import rank_world
    from .trainer import AgentConfig, Trainer
    opts, scene_args = build_parser().parse_known_args(sys.argv[1:] if argv is None else argv)
    pushes = push_schedule(opts)
    dyn = dynamics_randomization(opts)
    root = opts.asset_root or default_asset_root()
    agent_file, out_path, int_path = resolve_args(scene_args, root)
    model_files = resolve_model_files(scene_args, root)
    cfg = AgentConfig.from_json(agent_file)
    rank, world, local_rank = rank_world()
    group, device = None, opts.device
    if world > 1:
        import torch
        import torch.distributed as dist
        device = local_rank
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=torch.device("cuda", device))
        group = dist.group.WORLD
    os.makedirs(out_path, exist_ok=True)
    if int_path:
        os.makedirs(int_path, exist_ok=True)
    ckpt = rank_path(os.path.join(out_path, "agent0_checkpoint.pt"), rank)
    tr = Trainer(scene_args, cfg, root, opts.num_envs, window_steps=opts.window_steps, backend=opts.backend, seed=opts.seed, device=device,
                 log_path=os.path.join(out_path, "agent0_log.txt"), append_log=opts.resume is not None, process_group=group, model_files=model_files,
                 push_schedule=pushes, dynamics_randomization=dyn, latency_randomization=opts.rand_latency)
    if opts.resume:
        tr.load(rank_path(opts.resume, rank))
    try:
        while opts.max_iters is None or tr.iter < opts.max_iters:
            row = tr.iteration()
            if rank == 0:
                print("iteration %d: samples %d, Train_Return %.4f, Test_Return %.4f, %.2f s" % (row["Iteration"], row["Samples"], row["Train_Return"],
                                                                                                row["Test_Return"], row["Wall_Time"]), flush=True)
            if tr.iter % cfg["OutputIters"] == 0:
                tr.save(ckpt)
            if int_path and cfg["IntOutputIters"] > 0 and tr.iter % cfg["IntOutputIters"] == 0:
                tr.save(rank_path(os.path.join(int_path, "agent0_int_checkpoint_%010d.pt" % tr.iter), rank))
    except KeyboardInterrupt:
        pass
    tr.save(ckpt)
    tr.close()
    if rank == 0:
        print("checkpoint: %s (iteration %d)" % (ckpt, tr.iter))
    if group is not None:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
