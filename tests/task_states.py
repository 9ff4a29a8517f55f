"""Constructed inputs of the target_amp and heading_amp scenes' device code (dm_task.cuh through the step kernel's TASK glue, dm_task_reset_kernel
and dm_task_observe_kernel), built from oracle states so that every branch of the scene logic is reached on purpose rather than by a random
rollout.  tests/test_task_states_cpu.py checks in the oracle that each state takes its branch with every decision at least 10 % of its
threshold away from it; tests/test_task_branches_gpu.py compares the device with the oracle on them.

A state is an oracle prepared by `State.prepare`: the character airborne (no contacts, so the COM's horizontal velocity is the set root
velocity) or lying on the ground (fallen), the controller's clocks set so that the step has lasted a chosen time (need-new-action off, so one
update keeps the previous-action COM), the previous-action COM placed so that the COM's average velocity over the step is the chosen one, and
the task block (target, heading, speed, target timer) written directly.  Scene constants are overridden on the command line, which takes
precedence over --arg_file.

  target scene: COM velocity towards the target below / above tar_speed (enable_min_tar_vel on and off) and away from it; the root inside the
    success radius; the target within 1e-5 of the COM with success distance 0 (the td <= 1e-4 branch: unit vector 0); the target within 1e-5
    of the root (goal fallback); root headings in each quadrant and at +-pi; a fallen character; the root beyond tar_fail_dist with the target
    timer running and with it expiring on the same update (the redraw lands within max_target_dist < tar_fail_dist: no failure).
  heading scene: the timer expiring with a sharp turn (prob 1) and a Box-Muller turn (prob 0), a speed change (prob 1) and its clamp
    (tar_speed_min > tar_speed_max: the draw lies in (max, min] and the clamp returns max), tar_speed_min == tar_speed_max (no draw), the
    heading far past +-pi, avg_speed positive (below / above the target speed, enable_min_tar_vel on and off) and negative, fallen.
  timers (both scenes, 20-update launches): expiry on a chosen update, two expiries in one launch with timer_min == timer_max, a timer_max
    that is the double sum of k updates (the comparison meets it with equality)."""
import math
import os

import numpy as np

from tests import amp_states as A
from tests.parity_util import SnapLayout, random_policy_action

DT = 1.0 / 600.0
SCALE = 4.0
NJ = 15
LAY = SnapLayout(NJ)
CLK = LAY.scal                  # snapshot clocks: +8 ctrl, +9 init offset, +10 prev action, +11 need action, +12 timer, +13 timer max
CLOCK = {"ctrl": 8, "init_off": 9, "prev_action": 10, "need_action": 11, "timer": 12, "timer_max": 13}
K_COUNTER, K_RESET_SEEN = 12, 13
X_TAR_Y, X_HIT, X_HIT_TIME, X_GETUP = 16, 17, 18, 19

MINI = ["--motion_file", "data/datasets/test_clips_mini.txt"]
TARGET = MINI + ["--arg_file", "args/train_amp_target_humanoid3d_locomotion_args.txt"]
HEADING = MINI + ["--arg_file", "args/train_amp_heading_humanoid3d_locomotion_args.txt"]
SCENES = {"target": TARGET, "heading": HEADING}
STEP_UPDATES = 11               # the step has lasted 10 updates before the compared one: step_dur = 11 / 600 after it


# ---------------------------------------------------------------------------------------------------------------- oracle edits (shared with test_task_ext_gpu.py)
def set_clocks(o, **kw):
    s = o.get_snapshot()
    for k, v in kw.items():
        s[CLK + CLOCK[k]] = v
    o.set_snapshot(s)


def airborne(o, lift=2.0, vel=None):
    """the character lifted by `lift` m; with vel the joint velocities zeroed and every body moving with the root velocity vel (m/s)"""
    p, v = o.get_pose()
    p = p.copy(); p[1] += lift
    if vel is not None:
        v = np.zeros_like(v); v[0:3] = vel
    o.set_pose_vel(p, v)


def lying(o, seed):
    """brings the oracle's character to the ground: 1.5 s of wild random actions, then 0.5 s under the zero action, which keeps fall-contact
    bodies on the ground in every later update (checked by the callers against the oracle)"""
    off, scl, lo, hi = o.action_statics()
    rng = np.random.default_rng(seed)
    for _ in range(900):
        if o.need_new_action():
            o.set_action(random_policy_action(rng, off, scl, lo, hi, sigma=1.0))
        o.update(DT)
    o.set_action(-off)
    for _ in range(300):
        o.update(DT)


def load(core, e, o):
    """teacher forcing: the oracle's simulator snapshot and task block into environment e (the draw counter included; the reset counter kept)"""
    core.set_snapshot(e, o.get_snapshot())
    tb = core.task_state(e); ts = o.task_state()
    tb[0], tb[1] = ts["target_pos"][0], ts["target_pos"][2]
    tb[2:6] = [ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"]]
    tb[6:9] = ts["prev_action_com"]; tb[K_COUNTER] = o.task_counter()
    if o.goal_size == 4 and core.scene_name().startswith("Heading"):
        tb[X_GETUP] = o.getup_state()["timer"]
    elif o.goal_size == 4:
        ss = o.strike_state()
        tb[X_TAR_Y], tb[X_HIT], tb[X_HIT_TIME] = ss["target_height"], float(ss["hit"]), ss["hit_time"]
    core.set_task_state(e, tb)


def set_task(o, **kw):
    """the oracle's task block with some fields replaced (target as (x, z))"""
    ts = o.task_state()
    tp = ts["target_pos"].copy()
    if "target" in kw:
        tp[0], tp[2] = kw["target"]
    o.set_task_state(tp, kw.get("speed", ts["target_speed"]), kw.get("heading", ts["target_heading"]), kw.get("timer", ts["timer"]),
                     kw.get("timer_max", ts["timer_max"]), np.asarray(kw.get("prev_com", ts["prev_action_com"]), dtype=np.float64))


def root_xz(o):
    s = o.get_snapshot()
    return np.array([s[0], s[2]]) / SCALE


def heading_of_snapshot(s):
    """cKinTree::CalcHeading of the stored world -> base quaternion (x, y, z, w), as dm_task_observe_kernel computes it"""
    qx, qy, qz, qw = -s[3], -s[4], -s[5], s[6]
    return math.atan2(-2.0 * (qx * qz - qw * qy), 1.0 - 2.0 * (qy * qy + qz * qz))


# ---------------------------------------------------------------------------------------------------------------- scene constants
def scene_params(asset_root, args):
    """the scene constants of an argument list: defaults of cSceneTargetAMP / cSceneHeadingAMP, then --arg_file, then the command line"""
    p = dict(rand_target_time_min=0.2, rand_target_time_max=0.5, max_target_dist=10.0, target_succ_dist=0.5, tar_fail_dist=15.0, tar_speed=1.0,
             enable_min_tar_vel=False, pos_reward_scale=0.5, max_heading_turn_rate=0.15, sharp_turn_prob=0.01, speed_change_prob=0.02,
             tar_speed_min=1.0, tar_speed_max=5.0, vel_reward_scale=0.25)

    def take(tok):
        for i, t in enumerate(tok):
            k = t[2:]
            if t.startswith("--") and k in p and i + 1 < len(tok):
                v = tok[i + 1]
                p[k] = v.lower() == "true" if isinstance(p[k], bool) else float(v)
    with open(os.path.join(asset_root, args[args.index("--arg_file") + 1])) as f:
        take(f.read().split())
    take(args[:args.index("--arg_file")])
    return p


# ---------------------------------------------------------------------------------------------------------------- float64 restatement
def ref_reward(scene, p, tar, speed, heading, root, com, prev, step_dur, fallen, terms=None):
    """cSceneTargetAMP::CalcReward / cSceneHeadingAMP::CalcReward in float64 (SceneTargetAMP.cpp:3-80, SceneHeadingAMP.cpp:3-48); `terms`
    (a dict) receives the quantities the branches decide on"""
    t = {} if terms is None else terms
    if fallen:
        t["branch"] = "fallen"
        return 0.0
    if scene == "target":
        dx, dz = tar[0] - root[0], tar[1] - root[1]
        dsq = dx * dx + dz * dz
        t.update(dist_sq=dsq, fail=dsq > p["tar_fail_dist"] ** 2)
        if t["fail"]:
            t["branch"] = "fail"
            return 0.0
        pos_r = math.exp(-p["pos_reward_scale"] * dsq)
        if dsq < p["target_succ_dist"] ** 2:
            t["branch"] = "success"
            return 0.6 * pos_r + 0.4
        tx, tz = tar[0] - com[0], tar[1] - com[2]
        td = math.sqrt(tx * tx + tz * tz)
        t["td"] = td
        ux, uz = (tx / td, tz / td) if td > 1e-4 else (0.0, 0.0)
        avg = (ux * (com[0] - prev[0]) + uz * (com[2] - prev[2])) / step_dur
        t["avg"] = avg
        if avg < 0:
            t["branch"] = "away"
            return 0.6 * pos_r
        err = speed - avg
        if p["enable_min_tar_vel"]:
            err = max(err, 0.0)
        t["branch"] = "td0" if td <= 1e-4 else ("fast" if avg > speed else "slow")
        return 0.6 * pos_r + 0.4 * math.exp(-4.0 / (speed * speed) * err * err)
    avg = (math.cos(heading) * (com[0] - prev[0]) - math.sin(heading) * (com[2] - prev[2])) / step_dur
    t["avg"] = avg
    if not avg > 0.0:
        t["branch"] = "away"
        return 0.0
    err = speed - avg
    if p["enable_min_tar_vel"]:
        err = max(err, 0.0)
    t["branch"] = "fast" if avg > speed else "slow"
    return math.exp(-p["vel_reward_scale"] * err * err)


def ref_goal(scene, tar, speed, heading, root, root_heading):
    """cSceneTargetAMP::RecordGoal / cSceneHeadingAMP::RecordGoal in float64"""
    if scene == "target":
        rx, rz = tar[0] - root[0], tar[1] - root[1]
        d = math.hypot(rx, rz)
        if d <= 1e-4:
            return np.array([1.0, 0.0, d])
        c, s = math.cos(-root_heading), math.sin(-root_heading)
        return np.array([(c * rx + s * rz) / d, (-s * rx + c * rz) / d, d])
    th = heading - root_heading
    return np.array([math.cos(th), -math.sin(th), speed])


# ---------------------------------------------------------------------------------------------------------------- states
class State:
    """one constructed input.  scene: 'target' / 'heading'; extra: command-line overrides; kind: 'air' (airborne, root velocity `vel` along
    the reward direction, +- for away) or 'lying'; place: how the target / task block is set relative to the prepared character; expire: the
    target timer expires on this update of the comparison (0: it does not); branches: what the CPU test must see"""

    def __init__(self, name, scene, branches, extra=(), kind="air", speed=0.5, place="ahead", heading=None, expire=0, timer_max=None,
                 tar_heading=0.3, root_heading=0.9, tilt=None):
        self.name, self.scene, self.branches, self.extra, self.kind = name, scene, set(branches), list(extra), kind
        self.speed, self.place, self.heading, self.expire, self.timer_max = speed, place, heading, expire, timer_max
        self.tar_heading, self.root_heading, self.tilt = tar_heading, root_heading, tilt

    @property
    def args(self):
        return self.extra + SCENES[self.scene]

    def __repr__(self):
        return "%s/%s" % (self.scene, self.name)

    def prepare(self, o, p, stream, k=0):
        """the oracle `o` (built with self.args, its task stream `stream` = (seed, env) set) brought into this state; p: scene_params of
        self.args; k varies the clip time and the target direction between environments"""
        o.reset(0.2 + 0.07 * (k % 7), 0.0, 20.0, clip=0)
        if self.kind == "lying":
            s = _lying_snapshot(o)
            o.set_snapshot(s)
        s = A.with_heading(o, o.get_snapshot(), self.root_heading) if self.tilt is None else A.tilted(o, o.get_snapshot(), self.root_heading, self.tilt)
        o.set_snapshot(s)
        root = root_xz(o)
        # the reward direction: towards the target (target scene) or along the target heading (heading scene)
        if self.scene == "target":
            d = 6.0 if self.place in ("ahead", "expire_fail") else 4.0
            ang = 0.7 + 0.3 * k
            tar = root + d * np.array([math.cos(ang), math.sin(ang)])
            if self.place == "inside":
                tar = root + 0.25 * np.array([math.cos(ang), math.sin(ang)])
            elif self.place in ("beyond", "expire_fail"):
                tar = root + 16.5 * np.array([math.cos(ang), math.sin(ang)])
            u = (tar - root) / np.linalg.norm(tar - root)
        else:
            tar = root + 3.0 * np.array([math.cos(0.2 * k), math.sin(0.2 * k)])
            h = self.tar_heading + (40.0 * math.pi + 0.1 if self.place == "wound" else 0.0)
            if self.expire:   # the reward reads the heading the redraw gives: move along that one
                h = heading_redraw(o, p, stream, o.task_counter(), h, 1.0)[1]
            u = np.array([math.cos(h), -math.sin(h)])
        if self.kind == "air":
            airborne(o, vel=np.array([self.speed * u[0], 0.0, self.speed * u[1]]))
        sd = STEP_UPDATES * DT
        set_clocks(o, ctrl=1.0 + (STEP_UPDATES - 1) * DT, prev_action=1.0, init_off=0.0, need_action=0.0, timer=1.0 + (STEP_UPDATES - 1) * DT, timer_max=20.0)
        com_after = self._probe(o)
        prev = com_after.copy()
        prev[0] -= self.speed * u[0] * sd; prev[2] -= self.speed * u[1] * sd
        tmax = 20.0 if self.timer_max is None else self.timer_max
        timer = 0.5
        if self.expire:
            # the timer meets timer_max on update `expire` (half an update past it, or exactly with the double sum)
            timer = 0.5
            t = timer
            for _ in range(self.expire):
                t += DT
            tmax = t - 0.5 * DT
        kw = dict(target=tar, prev_com=prev, timer=timer, timer_max=tmax)
        if self.scene == "heading":
            kw["heading"] = self.tar_heading + (40.0 * math.pi + 0.1 if self.place == "wound" else 0.0)
            kw["speed"] = 1.0 if self.heading is None else self.heading
        if self.place in ("near_com", "near_root"):
            c = com_after if self.place == "near_com" else self._probe(o, root=True)
            kw["target"] = np.array([c[0] + 6e-6, c[2] - 7e-6]) if self.place == "near_com" else np.array([c[0] + 6e-6, c[1] - 7e-6])
        set_task(o, **kw)
        return o

    @staticmethod
    def _probe(o, root=False):
        """the COM (or the root x, z) after one update from the current state, with the target timer held off (no draw); the oracle is left
        as it was"""
        s, ts = o.get_snapshot(), o.task_state()
        o.set_task_state(ts["target_pos"], ts["target_speed"], ts["target_heading"], 0.0, 1e9, ts["prev_action_com"])
        o.update(DT)
        out = root_xz(o) if root else o.calc_com()
        o.set_snapshot(s)
        o.set_task_state(ts["target_pos"], ts["target_speed"], ts["target_heading"], ts["timer"], ts["timer_max"], ts["prev_action_com"])
        return out


_LYING = {}


def heading_redraw(o, p, stream, c0, old_heading, old_speed):
    """the heading scene's redraw on an expired timer (task_update), replayed on the draw stream (seed, env) from counter c0:
    (counter after it, new heading, new speed, branches taken)"""
    seed, env = stream
    k = [c0 + 2]                                                 # target distance and angle

    def u():
        k[0] += 1
        return o.u01(seed, env, k[0] - 1)
    br = set()
    if u() < p["sharp_turn_prob"]:
        h = old_heading + (-math.pi + u() * 2 * math.pi); br.add("sharp")
    else:
        u1 = u(); u2 = u()
        h = old_heading + p["max_heading_turn_rate"] * math.sqrt(-2.0 * math.log(1.0 - u1)) * math.cos(2 * math.pi * u2); br.add("normal")
    speed = old_speed
    if u() < p["speed_change_prob"]:
        br.add("speed_change")
        lo, hi = p["tar_speed_min"], p["tar_speed_max"]
        v = lo if lo == hi else lo + u() * (hi - lo)
        if lo == hi:
            br.add("speed_fixed")
        speed = min(max(v, lo), hi)
        if speed != v:
            br.add("speed_clamp")
    if p["rand_target_time_min"] != p["rand_target_time_max"]:
        u()
    return k[0], h, speed, br


def _lying_snapshot(o):
    """a character lying on the ground with fall-contact bodies in contact (built once per process)"""
    if "s" not in _LYING:
        lying(o, 17)
        _LYING["s"] = o.get_snapshot()
    return _LYING["s"]


QUADRANTS = [0.7, 2.3, -2.2, -0.8, math.pi, -math.pi]


def target_states():
    S = State
    out = [S("slow", "target", {"slow"}, speed=0.5),
           S("fast min-vel", "target", {"fast", "min_vel_on"}, speed=1.6),
           S("fast no min-vel", "target", {"fast", "min_vel_off"}, extra=["--enable_min_tar_vel", "false"], speed=1.6),
           S("slow no min-vel", "target", {"slow", "min_vel_off"}, extra=["--enable_min_tar_vel", "false"], speed=0.6),
           S("away", "target", {"away"}, speed=-0.8),
           S("inside", "target", {"success"}, place="inside", speed=0.3),
           S("target at the COM", "target", {"td0"}, extra=["--target_succ_dist", "0"], place="near_com", speed=0.0),
           S("target at the root", "target", {"goal_fallback"}, extra=["--target_succ_dist", "0"], place="near_root", speed=0.4),
           S("fallen", "target", {"fallen"}, kind="lying", speed=0.5),
           S("beyond", "target", {"fail"}, place="beyond", speed=0.5),
           S("beyond, redrawn", "target", {"expire_no_fail", "expire"}, place="expire_fail", speed=0.5, expire=1)]
    out += [S("heading %.4f" % h, "target", {"at_pi" if abs(h) == math.pi else "quadrant"}, root_heading=h, speed=0.7) for h in QUADRANTS]
    out += [S("tilted", "target", {"tilt"}, root_heading=0.4, tilt=math.radians(87.0), speed=0.7)]
    return out


def heading_states():
    S = State
    return [S("slow", "heading", {"slow"}, speed=0.5, heading=1.0),
            S("fast min-vel", "heading", {"fast", "min_vel_on"}, extra=["--enable_min_tar_vel", "true"], speed=2.0, heading=1.0),
            S("fast no min-vel", "heading", {"fast", "min_vel_off"}, speed=2.0, heading=1.0),
            S("away", "heading", {"away"}, speed=-0.7, heading=1.0),
            S("fallen", "heading", {"fallen"}, kind="lying", speed=0.5, heading=1.0),
            S("wound", "heading", {"wound", "slow"}, place="wound", speed=0.5, heading=1.0),
            S("sharp turn", "heading", {"expire", "sharp"}, extra=["--sharp_turn_prob", "1", "--speed_change_prob", "0"], expire=1, heading=1.0),
            S("normal turn", "heading", {"expire", "normal"}, extra=["--sharp_turn_prob", "0", "--speed_change_prob", "0"], expire=1, heading=1.0),
            S("speed change", "heading", {"expire", "normal", "speed_change"}, extra=["--sharp_turn_prob", "0", "--speed_change_prob", "1"], expire=1, heading=1.0),
            S("speed clamp", "heading", {"expire", "speed_clamp", "speed_change"},
              extra=["--sharp_turn_prob", "0", "--speed_change_prob", "1", "--tar_speed_min", "3", "--tar_speed_max", "2"], expire=1, heading=2.0),
            S("fixed speed", "heading", {"expire", "speed_fixed", "speed_change"},
              extra=["--sharp_turn_prob", "0", "--speed_change_prob", "1", "--tar_speed_min", "2.5", "--tar_speed_max", "2.5"], expire=1, heading=2.5)]


def all_states():
    return target_states() + heading_states()


# ---------------------------------------------------------------------------------------------------------------- 20-update launches
class Launch:
    """a 20-update launch from a new action: the character airborne with root velocity `vel` (m/s, x) so that the root moves between
    updates; the target timer expiring on update `first` (1-based) and, with fixed (timer_min == timer_max = `period` updates) timers, again
    every `period` updates; exact: timer_max is the double sum of the updates (the >= meets it with equality)"""

    def __init__(self, name, scene, first, period=None, exact=False, updates=20):
        self.name, self.scene, self.first, self.period, self.exact, self.updates = name, scene, first, period, exact, updates

    @property
    def args(self):
        if self.period is None:
            return SCENES[self.scene]
        t = repr(self.period * DT)
        return ["--rand_target_time_min", t, "--rand_target_time_max", t] + SCENES[self.scene]

    def __repr__(self):
        return "%s/%s" % (self.scene, self.name)

    def prepare(self, o, k=0):
        o.reset(0.25 + 0.05 * k, 0.0, 20.0, clip=0)
        airborne(o, lift=2.5, vel=np.array([2.5, 0.0, -1.0]))
        set_clocks(o, ctrl=0.0, prev_action=0.0, init_off=0.0, need_action=1.0, timer=0.0, timer_max=20.0)
        o.set_action(-o.action_statics()[0] + 0.05 * np.cos(np.arange(o.action_size) + k))
        t = 0.3
        T = t
        for _ in range(self.first):
            T += DT
        tmax = T if self.exact else T - 0.5 * DT
        set_task(o, timer=t, timer_max=tmax, prev_com=np.zeros(3))
        return o


def launches():
    return [Launch("expire on update 7", "target", 7), Launch("expire on update 13, exact", "target", 13, exact=True),
            Launch("three expiries, fixed timer", "target", 4, period=6), Launch("expire on update 7", "heading", 7),
            Launch("expire on update 19, exact", "heading", 19, exact=True), Launch("three expiries, fixed timer", "heading", 3, period=7),
            Launch("three policy steps", "target", 31, updates=60), Launch("three policy steps", "heading", 45, exact=True, updates=60)]
