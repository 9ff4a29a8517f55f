"""Constructed minibatches for the tensor-core learners' loss heads and input preparation (kernels/dm_learn.cu), and a float64 restatement of
the per-row rules those kernels implement.

The restatement is written from the reference's TF graph (R/learning/ppo_agent.py: _build_losses; pg_agent.py; tf_util.py: calc_bound_loss;
amp_agent.py: _build_losses), not from deepmimic_b200/learner.py, the torch backend, which is a second implementation of the same rules; the
CPU test checks that the two agree.  Every gradient is of the SUM over a step's rows (what the kernels write as dY; 1 / rows is the
optimiser's).

TF's gradient rules that decide a row's branch:
  * tf.minimum(x, y) passes the gradient to x where x <= y (ties go to x, the unclipped term);
  * tf.clip_by_value(t, lo, hi) passes it where lo <= t <= hi, bounds included;
  * calc_bound_loss: 0.5 sum_j (min(mu - lo, 0)^2 + max(mu - hi, 0)^2), so d/dmu = min(mu - lo, 0) + max(mu - hi, 0).

The constructions make each row's output exactly known: a "tagged trunk" (tagged_trunk) turns an integer tag in input column 0 into a one-hot
last hidden layer, exactly in fp16 and fp32, so that the output is b2 + W2[:, tag] (chosen fp16-exact) and the output layer's weight gradient
column `tag` is that row's dY alone.  Rows whose tag is BLANK have an all-zero last hidden layer (output b2, weight gradient untouched); rows
past the minibatch read zero inputs, which the trunk maps to tag 0, so column 0 of the weight gradient holds whatever the padding rows carry."""
import math

import numpy as np

F32, F16 = np.float32, np.float16
U32 = 2.0 ** -24        # fp32 unit roundoff
HALF_MAX = 65504.0      # the largest finite fp16
LOG_2PI_2 = 0.5 * math.log(2.0 * math.pi)
BLANK = -4              # a tag whose hidden layers are all zero
EPS = 0.2               # the reference agents' ratio_clip
LO, HI = -0.75, 0.625   # normalised action bounds of the actor constructions (fp16-exact)
SIGMA = 0.05            # the actor's exploration std (log-std log 0.05, as the reference's spin-kick agent)


# ---- the restatement (float64)
def gaussian_logp(norm_a, mu, logstd):
    """PGAgent's logp of the normalised action: sum_j -((a - mu) / sigma)^2 / 2 - log sigma - log(2 pi) / 2"""
    a, mu, ls = (np.asarray(v, dtype=np.float64) for v in (norm_a, mu, logstd))
    return (-0.5 * ((a - mu) / np.exp(ls)) ** 2 - ls - LOG_2PI_2).sum(axis=-1)


def ratio_clip_rule(adv, ratio, eps):
    """(active, clipped) per row, TF's rule applied in fp32 to a given fp32 ratio: l0 = adv ratio, l1 = adv clip(ratio, 1 - eps, 1 + eps);
    the surrogate's gradient reaches the row where l0 <= l1 (tf.minimum's tie) or 1 - eps <= ratio <= 1 + eps (tf.clip_by_value's);
    clipped: |ratio - 1| > eps (PPOAgent.clip_frac_tf)"""
    adv, r, e = F32(adv), F32(ratio), F32(eps)
    lo, hi = F32(1) - e, F32(1) + e
    inside = (r >= lo) & (r <= hi)
    l0, l1 = adv * r, adv * np.clip(r, lo, hi)
    return (l0 <= l1) | inside, np.abs(r - F32(1)) > e


def actor_rows(norm_a, mu, logstd, old_logp, adv, eps, bound_min, bound_max, ratio=None):
    """per row of the PPO actor: ratio (float64, or the given fp32 ratio), active, clipped, dY [rows, A] = d(-surrogate + bound loss) / dmu,
    surrogate, bound loss.  With `ratio` given the decisions and dY use it (the kernel's own state)"""
    mu, a = np.asarray(mu, np.float64), np.asarray(norm_a, np.float64)
    ls = np.asarray(logstd, np.float64)
    r64 = np.exp(gaussian_logp(a, mu, ls) - np.asarray(old_logp, np.float64))
    r = r64 if ratio is None else np.asarray(ratio, np.float64)
    active, clipped = ratio_clip_rule(adv, r, eps)
    adv64 = np.asarray(adv, np.float64)
    vmin, vmax = np.minimum(mu - np.asarray(bound_min, np.float64), 0.0), np.maximum(mu - np.asarray(bound_max, np.float64), 0.0)
    dy = np.where(active[:, None], -(adv64 * r)[:, None] * (a - mu) * np.exp(-2.0 * ls), 0.0) + vmin + vmax
    rc = np.clip(r, 1.0 - eps, 1.0 + eps)
    surr = np.minimum(adv64 * r, adv64 * rc)
    bound = 0.5 * (vmin ** 2 + vmax ** 2).sum(axis=-1)
    return dict(ratio=r64, active=active, clipped=clipped, dy=dy, surr=surr, bound=bound)


def actor_dy_bound(norm_a, mu, logstd, adv, ratio):
    """|dY_kernel - dY| per element given the kernel's ratio: the fp32 chain coef (a - mu) exp(-2 logstd) + vmin + vmax, about six roundings
    and expf's 2 ulp on the first term and two roundings on the violations (the bound terms are exact: fp16-exact mu and bounds), plus the
    hi + lo fp16 split of dY: 2^-22 |dY| + 2^-25 (fp16's subnormal spacing 2^-24, halved)"""
    a, mu = np.asarray(norm_a, np.float64), np.asarray(mu, np.float64)
    t = np.abs(np.asarray(adv, np.float64) * np.asarray(ratio, np.float64))[:, None] * np.abs(a - mu) * np.exp(-2.0 * np.asarray(logstd, np.float64))
    return 12 * U32 * (t + 1.0) + 2.0 ** -22 * (t + 2.0) + 2.0 ** -25


def ratio_bound(norm_a, mu, logstd, old_logp, ratio64):
    """|ratio_kernel - ratio|: the kernel sums logp in fp64 from fp32 terms -z^2/2 (z = (a - mu) / expf(logstd), IEEE division; each term
    within 6 u relative, expf's 2 ulp included), rounds lp - old_logp to fp32 (u |lp - old|) and takes expf (2 ulp): relative
    6 u sum_j (z_j^2 / 2) + u |log ratio| + 3 u, times ratio"""
    z2 = ((np.asarray(norm_a, np.float64) - np.asarray(mu, np.float64)) / np.exp(np.asarray(logstd, np.float64))) ** 2
    return ratio64 * (6 * U32 * 0.5 * z2.sum(axis=-1) + U32 * np.abs(np.log(ratio64)) + 3 * U32)


def critic_dy(out, target):
    """PPOAgent's critic loss 0.5 mean (target - V)^2 in the value normaliser's space: d/dV of the sum is V - target"""
    return np.asarray(out, np.float64) - np.asarray(target, np.float64)


def disc_rows(d_agent, d_expert):
    """AMPAgent's least-squares head (Peng et al. 2021, eq. 8) 0.5 (0.5 mean (d_e - 1)^2 + 0.5 mean (d_a + 1)^2): dY of the sum over rows,
    0.5 (d_a + 1) and 0.5 (d_e - 1), and the logged statistics: loss, acc_expert = mean(d_e > 0), acc_agent = mean(d_a < 0), the mean logits"""
    da, de = np.asarray(d_agent, np.float64), np.asarray(d_expert, np.float64)
    return dict(dy_agent=0.5 * (da + 1.0), dy_expert=0.5 * (de - 1.0),
                loss=0.5 * (0.5 * ((de - 1.0) ** 2).mean() + 0.5 * ((da + 1.0) ** 2).mean()),
                acc_expert=(de > 0).mean(), acc_agent=(da < 0).mean(), logit_expert=de.mean(), logit_agent=da.mean())


def prep_operand(s, mean, istd, clip):
    """the normalised, clipped input the trunk sees (float64; clip <= 0: no clip)"""
    x = (np.asarray(s, np.float64) - np.asarray(mean, np.float64)) * np.asarray(istd, np.float64)
    return x if clip <= 0 else np.clip(x, -clip, clip)


def prep_bound(x):
    """|fp16 operand - float64 value|: fp32 (s - mean) istd (2 u), fp16 rounding (2^-11 relative, 2^-25 absolute below 2^-14)"""
    return (2.0 ** -11 + 3 * U32) * np.abs(x) + 2.0 ** -25


def momentum_update(w, acc, g, lr, mom, wd):
    """TF MomentumOptimizer with the weight decay's gradient: acc' = mom acc + g + wd w, w' = w - lr acc' (float64)"""
    a = mom * np.asarray(acc, np.float64) + np.asarray(g, np.float64) + wd * np.asarray(w, np.float64)
    return np.asarray(w, np.float64) - lr * a, a


# ---- the tagged trunk
def tagged_trunk(in_dim, h0, h1):
    """(w0, b0, w1, b1) of a 2-layer ReLU trunk whose last hidden layer is one-hot in the integer tag of input column 0:
    h0_k = relu(t - k + 1), h1_j = relu(h0_j - 2 h0_{j+1} + h0_{j+2}) = [t == j] for integer t in [0, 2047] (every value an fp16-exact
    integer, every sum exact in fp32).  Units j >= h0 - 2 stay zero.  The tags a row can carry: 1 .. tag_count(h0, h1) - 1 (0 is the padding's)"""
    w0 = np.zeros((h0, in_dim), F32); w0[:, 0] = 1.0
    b0 = (1.0 - np.arange(h0)).astype(F32)
    w1 = np.zeros((h1, h0), F32)
    for j in range(min(h1, h0 - 2)):
        w1[j, j], w1[j, j + 1], w1[j, j + 2] = 1.0, -2.0, 1.0
    return w0, b0, w1, np.zeros(h1, F32)


def tag_count(h0, h1):
    return min(h1, h0 - 2, 2048)


def trunk_hidden(w0, b0, w1, b1, x):
    """float64 forward of the trunk on normalised inputs x [rows, in_dim]: the last hidden layer"""
    h = np.maximum(x @ w0.T.astype(np.float64) + b0, 0.0)
    return np.maximum(h @ w1.T.astype(np.float64) + b1, 0.0)


def _fp16_grid(v):
    """v rounded to fp16 and back (an output value the tagged trunk reproduces exactly)"""
    return np.asarray(v, F32).astype(F16).astype(F32)


# ---- the constructions
ACTOR_KINDS = ("inside+", "inside-", "hi clipped", "lo pessimistic", "hi pessimistic", "lo clipped", "adv 0", "ratio 1")
# (sign of the advantage, target ratio, expected active, expected clipped) of each kind at eps = 0.2
_ACTOR_KIND = {"inside+": (1, 1.05, True, False), "inside-": (-1, 0.95, True, False), "hi clipped": (1, 1.5, False, True),
               "lo pessimistic": (1, 0.5, True, True), "hi pessimistic": (-1, 1.5, True, True), "lo clipped": (-1, 0.5, False, True),
               "adv 0": (0, 1.3, True, True), "ratio 1": (1, 1.0, True, False)}
# normalised action means per component: below the lower bound, above the upper, inside, exactly on each bound
MU_KINDS = (("below", -1.25), ("above", 1.0), ("inside", 0.125), ("on lo", LO), ("on hi", HI))


def actor_case(A, rows, tags, seed, kinds=ACTOR_KINDS, edge=False):
    """a PPO actor minibatch over the tagged trunk.  rows: the minibatch's rows; tags: how many of them (the last ones) carry a tag, the rest
    are BLANK.  Tagged row i takes kind kinds[i % len] and its mu_j the MU_KINDS entry (i + j) % 5; BLANK rows have mu = 0 (inside the bounds)
    and kind "inside+".  edge: tagged rows target a ratio of exactly 1 + eps or 1 - eps (alternating) instead.
    Returns the per-sample arrays (one sample per minibatch row, idx = arange) and w2 [A, h1 >= tags + 1] as (tag -> mu) columns."""
    rng = np.random.default_rng(seed)
    tag = np.full(rows, BLANK, np.int64)
    tag[rows - tags:] = np.arange(1, tags + 1)
    kind = np.array(["inside+"] * rows, dtype=object)
    mu = np.zeros((rows, A), F32)
    for i, r in enumerate(range(rows - tags, rows)):
        kind[r] = ("edge hi" if i % 2 == 0 else "edge lo") if edge else kinds[i % len(kinds)]
        mu[r] = [MU_KINDS[(i + j) % len(MU_KINDS)][1] for j in range(A)]
    # edge rows: sigma = 1 / sqrt(2 pi) and |z| <= 0.04, so |logp| < 1e-3 and the fp32 old_logp puts the ratio within an ulp of its target
    logstd = np.full(A, -LOG_2PI_2 if edge else math.log(SIGMA), F32)
    z = np.clip(rng.standard_normal((rows, A)), -2.0, 2.0) * (0.02 if edge else 1.0)
    norm_a = (mu + np.exp(logstd) * z.astype(F32)).astype(F32)
    adv = np.empty(rows, F32)
    target = np.empty(rows)
    for r in range(rows):
        k = kind[r]
        if k.startswith("edge"):   # 1 +- eps moved by -2 .. 2 fp32 ulps, so that rows land on both sides of the fp32 bounds
            sign, target[r] = (1 if rng.random() < 0.5 else -1), (1.0 + EPS if k == "edge hi" else 1.0 - EPS) * (1.0 + ((r // 2) % 5 - 2) * 2.0 ** -23)
        else:
            sign, target[r] = _ACTOR_KIND[k][0], _ACTOR_KIND[k][1]
        if k == "ratio 1":
            norm_a[r] = mu[r]
        adv[r] = sign * rng.uniform(0.5, 4.0)
    old_logp = (gaussian_logp(norm_a, mu, logstd) - np.log(target)).astype(F32)
    return dict(tag=tag, kind=kind, mu=mu, norm_a=norm_a, adv=adv, old_logp=old_logp, logstd=logstd, target=target,
                bound_min=np.full(A, LO, F32), bound_max=np.full(A, HI, F32))


def output_layer(tag, values, h1, padding_value=0.0):
    """w2 [out, h1] whose column tag holds the output of the rows with that tag (fp16-exact values), b2 = 0; column 0 (the padding rows'
    tag) holds padding_value"""
    v = np.atleast_2d(np.asarray(values, F32).T).T if np.ndim(values) == 1 else np.asarray(values, F32)
    out = v.shape[1]
    w2 = np.zeros((out, h1), F32)
    for r in np.nonzero(tag >= 0)[0]:
        w2[:, tag[r]] = v[r]
    w2[:, 0] = padding_value
    assert np.array_equal(_fp16_grid(w2), w2), "the tagged outputs must be fp16-exact"
    return w2, np.zeros(out, F32)


def state_rows(tag, in_dim, seed):
    """raw states [rows, in_dim] with the tag in column 0 (the trunk ignores the other columns: its weights there are zero)"""
    s = np.random.default_rng(seed).standard_normal((len(tag), in_dim)).astype(F32)
    s[:, 0] = tag
    return s


def critic_case(rows, tags, seed):
    """a critic minibatch over the tagged trunk: value errors positive, negative and exactly zero (cycled over the tagged rows)"""
    rng = np.random.default_rng(seed)
    tag = np.full(rows, BLANK, np.int64)
    tag[rows - tags:] = np.arange(1, tags + 1)
    out = np.zeros(rows, F32)
    out[rows - tags:] = _fp16_grid(rng.uniform(-3.0, 3.0, tags))
    err = np.zeros(rows, F32)
    err[rows - tags:] = [(1.5, -2.25, 0.0)[i % 3] for i in range(tags)]
    err[:rows - tags] = _fp16_grid(rng.uniform(-1.0, 1.0, rows - tags))
    return dict(tag=tag, out=out, target=(out - err).astype(F32), err=err)


D_VALUES = (0.0, 1.0, -1.0, 2.5, -3.0, 0.5, -0.5, 4.0)


def disc_case(rows):
    """a discriminator minibatch over the tagged trunk: agent row r has tag 1 + r, expert row r tag 1 + rows + r; logits cycle through
    D_VALUES (0, +-1 and beyond), the expert side shifted by three so that both sides see every value"""
    tag_a, tag_e = 1 + np.arange(rows), 1 + rows + np.arange(rows)
    d_a = np.array([D_VALUES[r % len(D_VALUES)] for r in range(rows)], F32)
    d_e = np.array([D_VALUES[(r + 3) % len(D_VALUES)] for r in range(rows)], F32)
    return dict(tag_a=tag_a, tag_e=tag_e, d_a=d_a, d_e=d_e)
