"""Times the networks alone, CUDA events: the plain actor (4096 x 227 -> 1024 -> 512 -> 28, dm_mlp_forward), the gated task actor
(4096 x (226 + 3) -> 1024 -> 512 -> 28 with its gates, dm_mlp_forward_gated) and the AMP discriminator's reward (4096 x 226 -> 1024 -> 512 -> 1,
style reward and its blend with a task reward, dm_mlp_forward_style_reward) on the wgmma kernels, each against the fp32 torch network; then the
PPO critic of a rollout step (2 x 4096 rows [s_k; s'_k] x 227 -> 1024 -> 512 -> 1, un-normalised by the value normaliser) against the fp32 torch
critic, and the TD(lambda) return scan of a 600 x 4096 window (dm_td_lambda_returns) against a torch loop over the steps."""
import os, sys
import numpy as np
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch
from deepmimic_b200.capi import TensorCoreGatedMLP, TensorCoreMLP
rows, din, h0, h1, dout = int(os.environ.get("MLP_ROWS", "4096")), 227, 1024, 512, 28
rng = np.random.default_rng(0)
w0 = (rng.standard_normal((din, h0)) / np.sqrt(din)).astype(np.float32); w1 = (rng.standard_normal((h0, h1)) / np.sqrt(h0)).astype(np.float32); w2 = (rng.standard_normal((h1, dout)) / np.sqrt(h1)).astype(np.float32)
b0, b1, b2 = (rng.standard_normal(n).astype(np.float32) * 0.1 for n in (h0, h1, dout))
mean, std = rng.standard_normal(din).astype(np.float32), (0.5 + rng.random(din)).astype(np.float32)
mlp = TensorCoreMLP(w0, b0, w1, b1, w2, b2, in_mean=mean, in_std=std, in_clip=5.0, out_mean=np.zeros(dout, np.float32), out_std=np.ones(dout, np.float32), max_rows=rows)
x = torch.randn(rows, din, device="cuda"); out = torch.zeros(rows, dout, device="cuda"); noise = torch.zeros(rows, dout, device="cuda")
st = torch.cuda.current_stream()
tw = [torch.tensor(a, device="cuda") for a in (w0, b0, w1, b1, w2, b2, mean, std)]
def torch_actor():
    h = torch.clamp((x - tw[6]) / tw[7], -5, 5)
    h = torch.relu(h @ tw[0] + tw[1]); h = torch.relu(h @ tw[2] + tw[3]); return h @ tw[4] + tw[5]
def timeit(f, n=50):
    for _ in range(5): f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): f()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1000.0
t_tc = timeit(lambda: mlp.forward(x, out, noise=noise, stream=st.cuda_stream))
t_th = timeit(torch_actor)
ref = torch_actor(); torch.cuda.synchronize()
print("policy network, %d rows: wgmma kernels %.1f us per forward, fp32 torch actor %.1f us; max |diff| %.2e" % (rows, t_tc, t_th, (out - ref).abs().max().item()))

# the gated actor of the task scenes: goal 3, gate trunk 128, gate hidden 64
G, ds = 3, din - 1
lin = lambda a, b: ((rng.standard_normal((a, b)) / np.sqrt(a)).astype(np.float32), (rng.standard_normal(b) * 0.1).astype(np.float32))
actor = dict(hidden=[lin(ds + G, h0), lin(h0, h1)], mean=lin(h1, dout), gate_common=lin(G, 128),
             gates=[dict(hidden=lin(128, 64), scale=lin(64, h), bias=lin(64, h)) for h in (h0, h1)])
g_mean, g_std = rng.standard_normal(G).astype(np.float32), (0.5 + rng.random(G)).astype(np.float32)
gmlp = TensorCoreGatedMLP(actor, s_mean=mean[:ds], s_std=std[:ds], s_clip=5.0, g_mean=g_mean, g_std=g_std, g_clip=5.0, max_rows=rows)
xs, xg = x[:, :ds].contiguous(), torch.randn(rows, G, device="cuda")
T = lambda a: torch.tensor(a, device="cuda")
ta = {k: tuple(T(a) for a in v) for k, v in (("h0", actor["hidden"][0]), ("h1", actor["hidden"][1]), ("m", actor["mean"]), ("gc", actor["gate_common"]))}
tg = [{k: tuple(T(a) for a in g[k]) for k in ("hidden", "scale", "bias")} for g in actor["gates"]]
tn = [T(a) for a in (mean[:ds], std[:ds], g_mean, g_std)]
def torch_gated_actor():
    L = lambda v, wb: v @ wb[0] + wb[1]
    ns, ng = torch.clamp((xs - tn[0]) / tn[1], -5, 5), torch.clamp((xg - tn[2]) / tn[3], -5, 5)
    gc = torch.relu(L(ng, ta["gc"])); h = torch.cat([ns, ng], dim=-1)
    for w, g in zip((ta["h0"], ta["h1"]), tg):
        gh = torch.relu(L(gc, g["hidden"])); h = torch.relu(2.0 * torch.sigmoid(L(gh, g["scale"])) * L(h, w) + L(gh, g["bias"]))
    return L(h, ta["m"])
t_gtc = timeit(lambda: gmlp.forward(xs, xg, out, noise=noise, stream=st.cuda_stream))
t_gth = timeit(torch_gated_actor)
ref = torch_gated_actor(); torch.cuda.synchronize()
print("gated policy network, %d rows: wgmma kernels %.1f us per forward, fp32 torch actor %.1f us; max |diff| %.2e" % (rows, t_gtc, t_gth, (out - ref).abs().max().item()))

# the AMP discriminator's reward: normalise, 226 -> 1024 -> 512 -> 1 logit, style reward max(0, 1 - 0.25 (1 - d)^2), blend with a task reward
da = 226
disc = dict(hidden=[lin(da, h0), lin(h0, h1)], logit=lin(h1, 1))
dmlp = TensorCoreMLP(*disc["hidden"][0], *disc["hidden"][1], *disc["logit"], in_mean=mean[:da], in_std=std[:da], in_clip=5.0, max_rows=rows)
xa, task = x[:, :da].contiguous(), torch.rand(rows, device="cuda")
logit, style, reward = (torch.zeros(rows, device="cuda") for _ in range(3))
td = [T(a) for a in (*disc["hidden"][0], *disc["hidden"][1], *disc["logit"])]
def torch_disc_reward():
    h = torch.clamp((xa - tn[0]) / tn[1], -5, 5)
    h = torch.relu(h @ td[0] + td[1]); h = torch.relu(h @ td[2] + td[3]); d = (h @ td[4] + td[5])[:, 0]
    s = (1.0 - 0.25 * (1.0 - d) ** 2).clamp_min(0.0)
    return d, 0.5 * s + 0.5 * task
t_dtc = timeit(lambda: dmlp.style_reward(xa, reward, task_reward=task, task_lerp=0.5, logit=logit, style=style, stream=st.cuda_stream))
t_dth = timeit(torch_disc_reward)
ref_d, ref_r = torch_disc_reward(); torch.cuda.synchronize()
print("discriminator reward, %d rows: wgmma kernels %.1f us per forward, fp32 torch discriminator + reward ops %.1f us; max |logit diff| %.2e, max |reward diff| %.2e"
      % (rows, t_dtc, t_dth, (logit - ref_d).abs().max().item(), (reward - ref_r).abs().max().item()))

# the PPO critic of one rollout step: 2 x rows states [s_k; s'_k] -> 1024 -> 512 -> 1, value = 10 + 10 out (discount 0.95, rewards in [0, 1])
crit = dict(hidden=[lin(din, h0), lin(h0, h1)], out=lin(h1, 1))
cmlp = TensorCoreMLP(*crit["hidden"][0], *crit["hidden"][1], *crit["out"], in_mean=mean, in_std=std, in_clip=5.0, out_mean=[10.0], out_std=[10.0], max_rows=2 * rows)
x2, v2 = torch.randn(2 * rows, din, device="cuda"), torch.zeros(2 * rows, 1, device="cuda")
tcr = [T(a) for a in (*crit["hidden"][0], *crit["hidden"][1], *crit["out"])]
def torch_critic():
    h = torch.clamp((x2 - tw[6]) / tw[7], -5, 5)
    h = torch.relu(h @ tcr[0] + tcr[1]); h = torch.relu(h @ tcr[2] + tcr[3]); return 10.0 + 10.0 * (h @ tcr[4] + tcr[5])
t_ctc = timeit(lambda: cmlp.forward(x2, v2, stream=st.cuda_stream))
t_cth = timeit(torch_critic)
ref_v = torch_critic(); torch.cuda.synchronize()
print("critic, %d rows: wgmma kernels %.1f us per forward, fp32 torch critic %.1f us; max |value diff| %.2e" % (2 * rows, t_ctc, t_cth, (v2 - ref_v).abs().max().item()))

# the TD(lambda) return scan over a 600-step window
from deepmimic_b200.capi import td_lambda_returns
from deepmimic_b200.rollout import td_lambda_returns_host
sys.path.insert(0, os.path.join(REPO, "tests"))
from test_value_targets_cpu import synthetic_window
steps = 600
win = [torch.as_tensor(a).cuda() for a in synthetic_window(rng, steps, rows)]
ret, adv = torch.empty(steps, rows, device="cuda"), torch.empty(steps, rows, device="cuda")
ret2, adv2 = torch.empty_like(ret), torch.empty_like(adv)
t_k = timeit(lambda: td_lambda_returns(*win, 0.95, 0.95, 0.0, 20.0, ret, adv, stream=st.cuda_stream))
t_loop = timeit(lambda: td_lambda_returns_host(*win, 0.95, 0.95, 0.0, 20.0, ret2, adv2), n=5)
torch.cuda.synchronize()
print("TD(lambda) returns, %d x %d: return kernel %.1f us, torch loop over the steps %.1f us; max |return diff| %.2e" % (steps, rows, t_k, t_loop, (ret - ret2).abs().max().item()))
