"""Run a trained skill: the counterpart of the reference's `DeepMimic.py --arg_file args/run_*_args.txt`, without the viewer.

    python -m deepmimic_b200.run --arg_file args/run_humanoid3d_spinkick_args.txt [--model_files PATH] [--num_envs 64]
        [--record_motion K] [--render K [--render_size WxH] [--camera yaw,pitch,distance,height,fov_deg]] [--episode_time 20] [--backend tensor_core] [--seed 0] [--device 0] [--asset_root DIR]
        [--push_forces F1,F2,... [--push_body 0] [--push_time 2.0] [--push_duration 0.2]] [--dynamics_sweep KIND=V1,V2,...] [--latency_sweep S1,S2,...]
        [--pose_error] [--heading_course T:H:V,... | --target_course DX:DZ,...] [reference arguments ...]

--model_files (a reference TensorBundle prefix or a Trainer checkpoint, deepmimic_b200/model_files.py) and --output_path are read from the
argument list, the command line before the arg file, as deepmimic_b200.train reads its paths; --train_agents and --agent_files are accepted
and not needed.  The actor is the plain or the gated network, by the scene's goal size, as the Trainer chooses.  Every environment runs one
complete episode in test mode with exploration off, the loop of Trainer.evaluate; where the arguments set no episode time limit (the run_*
arg files: the reference's viewer runs until the character falls), an episode ends after --episode_time seconds (default 20).  Under
<output_path> (default "output"):
  run_log.txt          one row per environment: its return, its length in policy steps and its terminate code (0 time limit, 1 fail, 2 success)
  motion_<env>.txt     with --record_motion K, the first K environments' episodes as motion files (cMotion::Output, loop "none", one frame per
                       policy step and the terminal pose)
  render_<env>.png     with --render K, the first K environments' episodes as animated PNGs drawn by the device ray caster from the same
                       frames, each shown for one policy step (deepmimic_b200/render.py: --render_size, default 640x360, and --camera)
and a printed summary: the return's mean and standard deviation, the mean length and the fraction of episodes ended by Fail.  One GPU only.

Push robustness (--push_forces, the DeepMimic paper's test of a trained skill): environment e is pushed on body --push_body (default the root)
with the horizontal force of magnitude F[e % K] in N, for --push_duration seconds from --push_time seconds into its episode (defaults 0.2 and
2.0).  Each environment's direction is an angle drawn from --seed, the same every run.  run_log.txt then also has the columns Push_Force and
Push_Dir (radians, about the vertical axis from +x towards +z), and the summary one line per force: episodes, the fraction not ended by Fail
and the mean return.

Dynamics sweep (--dynamics_sweep KIND=V1,V2,..., KIND one of friction, kp, kd, torque_limit, mass): environment e runs with the factor V[e % K]
on that kind (DeepMimicBatchEnv.set_dynamics; for mass, every body's factor), the others 1.  run_log.txt then also has the column Dyn_<KIND>,
and the summary one line per value: episodes, the fraction not ended by Fail and the mean return.  It combines with --push_forces.

Latency sweep (--latency_sweep S1,S2,..., seconds): environment e runs with the control latency S[e % K], rounded to a whole 1/600 s update and
at most 19 updates (0.0317 s) (DeepMimicBatchEnv.set_action_latency): the PD targets of each action take effect that long after the policy
chose it.  run_log.txt then also has the column Latency (the rounded seconds), and the summary one line per value: episodes, the fraction not
ended by Fail and the mean return.  It combines with --push_forces and --dynamics_sweep.

Tracking error (--pose_error): how closely each episode followed its clip, in metres -- the mean over the non-root joints of the distance between
the simulated and the kinematic character's joint positions relative to the root, in each one's heading frame, over the poses the episode took
its actions in (BatchedCore.pose_error).  run_log.txt then also has the columns Pose_Err (phase-locked: frame i against the clip at the same
moment) and Pose_Err_DTW (after aligning the two motions by dynamic time warping, which forgives a skill that runs ahead of or behind its clip's
phase), the summary a line with the mean and standard deviation of both, and every per-force and per-value line both means.

Goal courses (DeepMimicBatchEnv.set_goal_course; one course for every environment, restarted at its reset):
  --heading_course T:H:V,...  (heading_amp, heading_amp_getup) commanded heading H (radians about the vertical axis, h = 0 along +x, the
      convention of --camera and Push_Dir) and speed V (m/s) from episode time T (s) on, linear in between; times increasing from >= 0.
      run_log.txt then also has Speed_Err (the mean |along-track speed - V| over the episode, m/s) and Cross_Speed (the mean |cross-track
      speed|), and the summary a line with their means and the fraction not ended by Fail.
  --target_course DX:DZ,...   (target_amp) waypoints in metres from where the character starts, each reached within the scene's success
      radius, in order.  run_log.txt then also has Waypoints (the number reached) and Course_Time (the episode time at which the last one was
      reached, nan if never), and the summary a line with the mean reached, the fraction that reached all and their mean time.
At most 16 points.  Both combine with the push, dynamics and latency sweeps, whose per-value lines then carry the course's means, and with
--render, whose frames draw the recorded goal (the point 1.5 m ahead along the commanded heading, or the waypoint) as a green sphere on the
ground."""
import argparse
import os
import sys

from .render import add_view_options
from .train import arg_table, first_arg, resolve_model_files


def build_parser():
    ap = argparse.ArgumentParser(prog="python -m deepmimic_b200.run", description=__doc__.split("\n\n")[0], allow_abbrev=False)
    ap.add_argument("--asset_root", default=None, help="the reference's data / args tree (default: the bundled asset archive)")
    ap.add_argument("--num_envs", type=int, default=64, help="environments, one episode each")
    ap.add_argument("--record_motion", type=int, default=0, metavar="K", help="write the first K environments' episodes as motion files")
    ap.add_argument("--render", type=int, default=0, metavar="K", help="write the first K environments' episodes as animated PNGs")
    add_view_options(ap)
    ap.add_argument("--backend", default="tensor_core", choices=("tensor_core", "torch"))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--episode_time", type=float, default=20.0,
                    help="test-mode episode limit in seconds for arguments that set none (the run_* arg files; default 20, the train_* files' limit)")
    ap.add_argument("--push_forces", type=parse_forces, default=None, metavar="F1,F2,...",
                    help="push-robustness sweep: horizontal push magnitudes in N (>= 0), environment e gets F[e %% K]")
    ap.add_argument("--push_body", type=int, default=0, help="body pushed in the sweep (default 0, the root)")
    ap.add_argument("--push_time", type=float, default=2.0, help="episode time of the push in seconds (default 2.0)")
    ap.add_argument("--push_duration", type=float, default=0.2, help="length of the push in seconds (default 0.2)")
    ap.add_argument("--dynamics_sweep", type=parse_dynamics_sweep, default=None, metavar="KIND=V1,V2,...",
                    help="dynamics sweep: factors on friction, kp, kd, torque_limit or mass, environment e gets V[e %% K]")
    ap.add_argument("--latency_sweep", type=parse_latency_sweep, default=None, metavar="S1,S2,...",
                    help="latency sweep: control latencies in s (whole 1/600 s updates, at most 0.0317 s), environment e gets S[e %% K]")
    ap.add_argument("--pose_error", action="store_true",
                    help="score each episode's tracking of its clip: phase-locked and time-warped joint-position error in metres")
    course = ap.add_mutually_exclusive_group()
    course.add_argument("--heading_course", type=parse_heading_course, default=None, metavar="T:H:V,...",
                        help="heading scenes: commanded heading H (rad) and speed V (m/s) from episode time T (s), linear in between")
    course.add_argument("--target_course", type=parse_target_course, default=None, metavar="DX:DZ,...",
                        help="target scene: waypoints in m from the start position, visited in order")
    return ap


MAX_COURSE_POINTS = 16
MARKER_HEIGHT, MARKER_RADIUS = 0.1, 0.1   # m: the goal drawn by --render with a course, a sphere resting on the ground


def _parse_points(text, width, form):
    """comma-separated points of `width` colon-separated finite numbers: [K, width] lists, 1 <= K <= MAX_COURSE_POINTS"""
    import math
    try:
        pts = [[float(x) for x in p.split(":")] for p in text.split(",")]
    except ValueError:
        raise argparse.ArgumentTypeError("need %s, got %r" % (form, text))
    if any(len(p) != width for p in pts) or not 1 <= len(pts) <= MAX_COURSE_POINTS:
        raise argparse.ArgumentTypeError("need 1 to %d points %s, got %r" % (MAX_COURSE_POINTS, form, text))
    if any(not math.isfinite(x) for p in pts for x in p):
        raise argparse.ArgumentTypeError("course values must be finite, got %r" % text)
    return pts


def parse_heading_course(text):
    """T:H:V,...: [K, 3] rows (episode time s, heading rad, speed m/s), times strictly increasing from >= 0, speeds >= 0"""
    pts = _parse_points(text, 3, "T:H:V,... (seconds, radians, m/s)")
    if pts[0][0] < 0.0 or any(b[0] <= a[0] for a, b in zip(pts, pts[1:])):
        raise argparse.ArgumentTypeError("heading course times must increase from >= 0, got %r" % text)
    if any(p[2] < 0.0 for p in pts):
        raise argparse.ArgumentTypeError("heading course speeds must be >= 0, got %r" % text)
    return pts


def parse_target_course(text):
    """DX:DZ,...: [K, 2] waypoints in metres from the start position"""
    return _parse_points(text, 2, "DX:DZ,... (metres)")


def course_markers(rec, length):
    """[length + 1, 4] marker rows (x, MARKER_HEIGHT, z, MARKER_RADIUS) of one environment's episode frames from its course records [T, 4]:
    frame f > 0 draws the record of step f - 1 (the step that ended in it), frame 0 that of step 0"""
    import numpy as np
    rec = np.asarray(rec, dtype=np.float64)
    idx = np.maximum(np.arange(length + 1) - 1, 0)
    m = np.empty((length + 1, 4), dtype=np.float32)
    m[:, 0], m[:, 1], m[:, 2], m[:, 3] = rec[idx, 0], MARKER_HEIGHT, rec[idx, 1], MARKER_RADIUS
    return m


DYNAMICS_KINDS = ("friction", "kp", "kd", "torque_limit", "mass")


def parse_dynamics_sweep(text):
    """KIND=V1,V2,...: (kind, [values]); finite values >= 0, > 0 for mass"""
    kind, _, vals = text.partition("=")
    if kind not in DYNAMICS_KINDS:
        raise argparse.ArgumentTypeError("need KIND=V1,V2,... with KIND one of %s, got %r" % (", ".join(DYNAMICS_KINDS), text))
    try:
        v = [float(x) for x in vals.split(",")]
    except ValueError:
        raise argparse.ArgumentTypeError("need comma-separated numbers after %s=, got %r" % (kind, text))
    if not v or any(not (x >= 0.0) or x == float("inf") for x in v) or (kind == "mass" and min(v) <= 0.0):
        raise argparse.ArgumentTypeError("%s factors must be finite and %s, got %r" % (kind, "> 0" if kind == "mass" else ">= 0", text))
    return kind, v


def dynamics_plan(sweep, num_envs):
    """the sweep's per-environment factor [N] (environment e gets values[e % K])"""
    import numpy as np
    kind, values = sweep
    return np.asarray([values[e % len(values)] for e in range(num_envs)], dtype=np.float32)


def parse_latency_sweep(text):
    """S1,S2,...: the latencies in seconds, each rounded to a whole update in [0, 19]; returns the rounded seconds"""
    from .capi import UPDATE_DT, UPDATES_PER_ACTION, latency_updates
    try:
        v = [float(x) for x in text.split(",")]
    except ValueError:
        raise argparse.ArgumentTypeError("need comma-separated latencies in seconds, got %r" % text)
    try:
        return [latency_updates(x, UPDATES_PER_ACTION, "--latency_sweep") * UPDATE_DT for x in v]
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e))


def parse_forces(text):
    try:
        forces = [float(x) for x in text.split(",")]
    except ValueError:
        raise argparse.ArgumentTypeError("need comma-separated numbers, got %r" % text)
    if not forces or any(not (f >= 0.0) or f == float("inf") for f in forces):
        raise argparse.ArgumentTypeError("push forces must be finite and >= 0, got %r" % text)
    return forces


def push_plan(forces, num_envs, seed):
    """the sweep's pushes: magnitude [N] (environment e gets forces[e % K]), direction [N] (an angle in [0, 2 pi) about the vertical axis per
    environment, drawn from seed) and the world-axes force [N, 3] float32"""
    import numpy as np
    mag = np.asarray([forces[e % len(forces)] for e in range(num_envs)], dtype=np.float64)
    ang = np.random.default_rng(seed).uniform(0.0, 2.0 * np.pi, num_envs)
    force = np.stack([mag * np.cos(ang), np.zeros(num_envs), mag * np.sin(ang)], axis=1).astype(np.float32)
    return mag, ang, force


def write_episode_motions(path_fmt, ep, count, frame_dur):
    """motion files of the first `count` environments of run_episodes(pose_envs >= count)'s result `ep`: path_fmt % env; returns the paths"""
    from .formats import write_motion
    from .rollout import episode_motion
    lengths = ep["lengths"].cpu().tolist()
    paths = []
    for e in range(count):
        frames = episode_motion(ep["poses"], ep["end_poses"], e, int(lengths[e]))
        write_motion(path_fmt % e, frames, [frame_dur] * frames.shape[0], loop="none")
        paths.append(path_fmt % e)
    return paths


def write_episode_renders(path_fmt, ep, count, frame_dur, core, camera=None, size=(640, 360)):
    """animated PNGs of the first `count` environments of run_episodes(pose_envs >= count)'s result `ep`, the frames of write_episode_motions
    drawn as core's character, with the goal of each frame (course_markers) when ep has course records: path_fmt % env; returns the paths"""
    from .render import write_pose_apng
    from .rollout import episode_motion
    lengths = ep["lengths"].cpu().tolist()
    paths = []
    for e in range(count):
        frames = episode_motion(ep["poses"], ep["end_poses"], e, int(lengths[e]))
        if "course" in ep:
            marks = course_markers(ep["course"][:, e].cpu().numpy(), int(lengths[e]))
            write_pose_apng(core, path_fmt % e, frames, [frame_dur] * frames.shape[0], camera, size, markers=marks)
        else:
            write_pose_apng(core, path_fmt % e, frames, [frame_dur] * frames.shape[0], camera, size)
        paths.append(path_fmt % e)
    return paths


def main(argv=None):
    import numpy as np
    from .assets import asset_root as default_asset_root
    from .sharding import rank_world
    opts, scene_args = build_parser().parse_known_args(sys.argv[1:] if argv is None else argv)
    if rank_world()[1] > 1:
        raise SystemExit("run: one GPU only; start it without torchrun")
    if opts.num_envs < 1 or not 0 <= opts.record_motion <= opts.num_envs or not 0 <= opts.render <= opts.num_envs:
        raise SystemExit("run: need --num_envs >= 1, 0 <= --record_motion <= --num_envs and 0 <= --render <= --num_envs")
    if opts.push_forces is not None and not (opts.push_duration >= 0.0 and np.isfinite(opts.push_duration) and np.isfinite(opts.push_time)):
        raise SystemExit("run: need a finite --push_time and a finite --push_duration >= 0")
    root = opts.asset_root or default_asset_root()
    table = arg_table(scene_args, root, "run")
    out_path = first_arg(table, "output_path") or "output"
    model_files = resolve_model_files(scene_args, root, "run")
    if model_files is None:
        raise SystemExit("run: no --model_files in the arguments or the arg file")
    from .model_files import model_file_kind
    try:
        model_file_kind(model_files)
    except FileNotFoundError as e:
        raise SystemExit("run: %s" % e)
    import torch
    from .env import DeepMimicBatchEnv
    from .formats import TableLog
    from .model_files import load_model_files
    from .rollout import BatchedRollout, run_episodes
    if not (first_arg(table, "time_end_lim_max") or first_arg(table, "time_lim_max")):
        # the reference's viewer runs an episode until the character falls; one complete episode per environment needs an end
        scene_args = scene_args + ["--time_end_lim_min", repr(opts.episode_time), "--time_end_lim_max", repr(opts.episode_time)]
    env = DeepMimicBatchEnv(scene_args, opts.num_envs, root, device=opts.device, seed=opts.seed)
    env.set_mode(1)
    env.reset(True)
    if opts.push_forces is not None:
        N = opts.num_envs
        mag, ang, force = push_plan(opts.push_forces, N, opts.seed)
        env.set_pushes(np.full(N, opts.push_body, dtype=np.int32), force, np.full(N, opts.push_time), np.full(N, opts.push_duration))
    if opts.dynamics_sweep is not None:
        kind, fac = opts.dynamics_sweep[0], dynamics_plan(opts.dynamics_sweep, opts.num_envs)
        env.set_dynamics(**{kind: (np.repeat(fac[:, None], env._core.dims.num_joints, axis=1) if kind == "mass" else fac)})
    if opts.latency_sweep is not None:
        lat = np.asarray([opts.latency_sweep[e % len(opts.latency_sweep)] for e in range(opts.num_envs)])
        env.set_action_latency(lat)
    course = opts.heading_course or opts.target_course
    if course is not None:
        kind = int(env._core.task_params()[0][0])   # 1 target_amp, 2 heading_amp, 3 heading_amp_getup
        if (opts.heading_course is not None and kind not in (2, 3)) or (opts.target_course is not None and kind != 1):
            raise SystemExit("run: --%s needs the %s scene, not %s" % ("heading_course" if opts.heading_course is not None else "target_course",
                                                                     "heading_amp or heading_amp_getup" if opts.heading_course is not None
                                                                     else "target_amp", env.get_name()))
        env.set_goal_course(np.asarray(course, dtype=np.float64))
    ro = BatchedRollout(env, exp_rate=0.0, seed=opts.seed, backend=opts.backend)
    norms = dict(s_norm=ro.s_norm, a_norm=ro.a_norm, **(dict(g_norm=ro.g_norm) if ro.goal_size > 0 else {}))
    try:
        load_model_files(model_files, ro.policy, norms)
    except ValueError as e:
        raise SystemExit("run: %s" % e)
    ep = run_episodes(ro, pose_envs=max(opts.record_motion, opts.render), pose_error=opts.pose_error, course=course is not None)
    torch.cuda.synchronize(env.device)
    ret, length, term = (ep[k].cpu().numpy() for k in ("returns", "lengths", "terminate"))
    if opts.pose_error:
        perr, perr_dtw = ep["pose_err"].cpu().numpy(), ep["pose_err_dtw"].cpu().numpy()
    course_cols = {}
    if opts.heading_course is not None:
        course_cols = dict(Speed_Err=ep["speed_err"].cpu().numpy(), Cross_Speed=ep["cross_speed"].cpu().numpy())
    elif opts.target_course is not None:
        course_cols = dict(Waypoints=ep["waypoints"].cpu().numpy(), Course_Time=ep["course_time"].cpu().numpy())

    def course_means(sel):
        if opts.heading_course is not None:
            return ", speed error %.4f m/s, cross-track speed %.4f m/s" % (float(np.mean(course_cols["Speed_Err"][sel])),
                                                                           float(np.mean(course_cols["Cross_Speed"][sel])))
        if opts.target_course is not None:
            wp, ct = course_cols["Waypoints"][sel], course_cols["Course_Time"][sel]
            done = np.isfinite(ct)
            return ", waypoints %.2f of %d, all reached %.3f in %s s" % (float(np.mean(wp)), len(course), float(np.mean(done)),
                                                                       "%.3f" % float(np.mean(ct[done])) if done.any() else "nan")
        return ""
    err_means = lambda sel: ((", pose error %.4f m, DTW %.4f m" % (float(np.mean(perr[sel])), float(np.mean(perr_dtw[sel]))))
                             if opts.pose_error else "") + course_means(sel)
    os.makedirs(out_path, exist_ok=True)
    log = TableLog(os.path.join(out_path, "run_log.txt"))
    for e in range(opts.num_envs):
        for k, v in (("Env", e), ("Return", float(ret[e])), ("Length", int(length[e])), ("Terminate", int(term[e]))):
            log.log_tabular(k, v)
        if opts.push_forces is not None:
            log.log_tabular("Push_Force", float(mag[e]))
            log.log_tabular("Push_Dir", float(ang[e]))
        if opts.dynamics_sweep is not None:
            log.log_tabular("Dyn_" + kind, opts.dynamics_sweep[1][e % len(opts.dynamics_sweep[1])])
        if opts.latency_sweep is not None:
            log.log_tabular("Latency", float(lat[e]))
        if opts.pose_error:
            log.log_tabular("Pose_Err", float(perr[e]))
            log.log_tabular("Pose_Err_DTW", float(perr_dtw[e]))
        for k, v in course_cols.items():
            log.log_tabular(k, float(v[e]))
        log.dump_tabular()
    log.close()
    print("%s, %d episodes: return %.4f +- %.4f, length %.1f policy steps, ended by Fail %.3f" % (model_files, opts.num_envs, float(np.mean(ret)),
                                                                                              float(np.std(ret)), float(np.mean(length)), float(np.mean(term == 1))))
    if opts.pose_error:
        print("pose error %.4f +- %.4f m, time-warped %.4f +- %.4f m" % (float(np.mean(perr)), float(np.std(perr)), float(np.mean(perr_dtw)),
                                                                     float(np.std(perr_dtw))))
    if course is not None:
        print("%s course of %d points: %d episodes, not ended by Fail %.3f%s" % ("heading" if opts.heading_course is not None else "target",
                                                                             len(course), opts.num_envs, float(np.mean(term != 1)),
                                                                             course_means(np.ones(opts.num_envs, dtype=bool))))
    if opts.push_forces is not None:
        for f in opts.push_forces:
            sel = mag == f
            print("push %g N on body %d at %g s for %g s: %d episodes, not ended by Fail %.3f, return %.4f%s" % (
                f, opts.push_body, opts.push_time, opts.push_duration, int(sel.sum()), float(np.mean(term[sel] != 1)), float(np.mean(ret[sel])),
                err_means(sel)))
    if opts.dynamics_sweep is not None:
        for v in opts.dynamics_sweep[1]:
            sel = fac == np.float32(v)
            print("%s x %g: %d episodes, not ended by Fail %.3f, return %.4f%s" % (kind, v, int(sel.sum()), float(np.mean(term[sel] != 1)),
                                                                                    float(np.mean(ret[sel])), err_means(sel)))
    if opts.latency_sweep is not None:
        for v in dict.fromkeys(opts.latency_sweep):
            sel = lat == v
            print("latency %.4f s (%d updates): %d episodes, not ended by Fail %.3f, return %.4f%s" % (
                v, round(v / env.UPDATE_DT), int(sel.sum()), float(np.mean(term[sel] != 1)), float(np.mean(ret[sel])), err_means(sel)))
    if opts.record_motion:
        paths = write_episode_motions(os.path.join(out_path, "motion_%d.txt"), ep, opts.record_motion,
                                      env.get_updates_per_action() * env.UPDATE_DT)
        print("motion files: %s .. %s" % (paths[0], paths[-1]))
    if opts.render:
        paths = write_episode_renders(os.path.join(out_path, "render_%d.png"), ep, opts.render, env.get_updates_per_action() * env.UPDATE_DT,
                                      env._core, opts.camera, opts.render_size)
        print("renders: %s .. %s" % (paths[0], paths[-1]))
    out = dict(returns=ret, lengths=length, terminate=term)
    if opts.pose_error:
        out.update(pose_err=perr, pose_err_dtw=perr_dtw)
    out.update({k.lower(): v for k, v in course_cols.items()})
    return out


if __name__ == "__main__":
    main()
