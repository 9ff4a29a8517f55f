"""Model files (--model_files): a trained policy to run or to start training from, read into the rollout's torch modules and normalisers.

Two kinds of file are read:
  a reference TensorBundle prefix (<prefix>.index + <prefix>.data-*, e.g. data/policies/humanoid3d/humanoid3d_spinkick.ckpt, written by the
    reference's tf.train.Saver): the actor (tf_checkpoint.load_actor), the critic when the bundle has one (tf_checkpoint.load_critic), and the
    normalisers s_norm, g_norm, a_norm and val_norm with their sample counts when the bundle holds them.  The critic's names and the counts
    are readings of the reference's scopes that have not been checked against a checkpoint it wrote.
  a Trainer checkpoint (.pt, Trainer.save): the networks (actor, critic and, for an AMP agent, the discriminator) and every normaliser with its
    count.

load_model_files refuses a file whose networks do not fit the modules it is given, naming the field: the state, goal or action size, a plain
against a gated network, or the hidden widths.  What the file lacks stays as initialised, with a warning."""
import os
import warnings

import numpy as np

_NORM_FIELDS = ("mean", "mean_sq", "std")


def model_file_kind(path):
    """"checkpoint" for a Trainer checkpoint file, "bundle" for a TensorBundle prefix; FileNotFoundError naming the path otherwise"""
    if os.path.isfile(path):
        return "checkpoint"
    if os.path.isfile(path + ".index"):
        return "bundle"
    raise FileNotFoundError("model file %s not found (neither a checkpoint file nor a TensorBundle prefix with %s.index)" % (path, path))


def _module_signature(net, head):
    """(network kind, goal size, state size, output size, hidden widths, gate widths) of an actor (rollout.build_policy /
    build_gated_policy, head = its mean layer) or a critic (rollout.build_critic, head = its out layer)"""
    gated = hasattr(net, "gate_common")
    G = net.gate_common.in_features if gated else 0
    gates = (net.gate_common.out_features, net.gate_hidden[0].out_features) if gated else ()
    return ("gated" if gated else "plain", G, net.hidden[0].in_features - G, head.out_features, tuple(l.out_features for l in net.hidden), gates)


def _bundle_signature(a, head):
    """the same signature of a tf_checkpoint.load_actor (head "mean") or load_critic (head "out") dict"""
    gated = "gate_common" in a
    G = a["gate_common"][0].shape[0] if gated else 0
    gates = (a["gate_common"][0].shape[1], a["gates"][0]["hidden"][0].shape[1]) if gated else ()
    return ("gated" if gated else "plain", G, a["hidden"][0][0].shape[0] - G, a[head][0].shape[1], tuple(w.shape[1] for w, _ in a["hidden"]), gates)


def _state_dict_signature(sd):
    """the same signature of a policy module's state_dict"""
    gated = "gate_common.weight" in sd
    G = sd["gate_common.weight"].shape[1] if gated else 0
    gates = (sd["gate_common.weight"].shape[0], sd["gate_hidden.0.weight"].shape[0]) if gated else ()
    widths, i = [], 0
    while "hidden.%d.weight" % i in sd:
        widths.append(sd["hidden.%d.weight" % i].shape[0]); i += 1
    return ("gated" if gated else "plain", G, sd["hidden.0.weight"].shape[1] - G, sd["mean.weight"].shape[0], tuple(widths), gates)


def _check_signature(path, what, have, want):
    """what: "actor" or "critic"; the first differing field is named"""
    fields = ("network", "goal size", "state size", "action size" if what == "actor" else "output size", "hidden widths", "gate widths")
    for name, h, w in zip(fields, have, want):
        if h != w:
            raise ValueError("model file %s: its %s%s is %s, this scene's %s needs %s" % (path, "" if what == "actor" else "critic's ", name, h, what, w))


def _check_state_dict(path, what, module, sd):
    """every parameter of `module` in sd with the same shape"""
    for k, v in module.state_dict().items():
        if k not in sd:
            raise ValueError("model file %s: %s.%s is missing" % (path, what, k))
        if tuple(sd[k].shape) != tuple(v.shape):
            raise ValueError("model file %s: %s.%s has shape %s, this scene's %s needs %s" % (path, what, k, tuple(sd[k].shape), what, tuple(v.shape)))


def _check_norm(path, name, norm, mean):
    if np.asarray(mean).size != norm.mean.numel():
        raise ValueError("model file %s: %s has %d entries, this scene's needs %d" % (path, name, np.asarray(mean).size, norm.mean.numel()))


def _note(notes, msg):
    warnings.warn(msg)
    notes.append(msg)


def load_model_files(path, policy, norms, critic=None, disc=None):
    """Reads `path` (model_file_kind) into the actor `policy`, the normalisers `norms` ({name: rollout.DeviceNormalizer}, names s_norm,
    g_norm, a_norm, val_norm, amp_norm; those the file lacks are kept), the critic and the discriminator (either may be None: not loaded).
    Every size is checked before anything is written.  A loaded normaliser takes the file's statistics and its pending sums are cleared.
    Returns dict(kind, counts = {loaded normaliser: the file's sample count, or None when the file has none}, notes = what stayed as
    initialised, each also given as a warning)."""
    import torch
    kind = model_file_kind(path)
    notes, counts = [], {}
    if kind == "bundle":
        from .rollout import load_actor_weights, load_critic_weights
        from .tf_checkpoint import list_entries, load_actor, load_critic
        actor = load_actor(path)
        _check_signature(path, "actor", _bundle_signature(actor, "mean"), _module_signature(policy, policy.mean))
        has_critic = "agent/main/critic/dense/kernel" in list_entries(path)
        crit = load_critic(path) if critic is not None and has_critic else None
        if crit is not None:
            _check_signature(path, "critic", _bundle_signature(crit, "out"), _module_signature(critic, critic.out))
        stats = {}
        for name, src in (("s_norm", actor), ("g_norm", actor), ("a_norm", actor), ("val_norm", crit or {})):
            if name in norms and name + "_mean" in src:
                _check_norm(path, name, norms[name], src[name + "_mean"])
                stats[name] = src
        load_actor_weights(policy, actor)
        if crit is not None:
            load_critic_weights(critic, crit)
        elif critic is not None:
            _note(notes, "model file %s has no critic: the critic stays as initialised" % path)
        for name, src in stats.items():
            n = norms[name]
            n.set_mean_std(src[name + "_mean"], src[name + "_std"])
            n.new_count = 0; n.new_sum.zero_(); n.new_sum_sq.zero_()
            counts[name] = int(np.asarray(src[name + "_count"]).reshape(-1)[0]) if name + "_count" in src else None
    else:
        s = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(s, dict) or "nets" not in s or "norms" not in s:
            raise ValueError("model file %s is not a Trainer checkpoint (no nets / norms)" % path)
        nets = s["nets"]
        _check_signature(path, "actor", _state_dict_signature(nets["actor"]), _module_signature(policy, policy.mean))
        _check_state_dict(path, "actor", policy, nets["actor"])
        if critic is not None:
            _check_state_dict(path, "critic", critic, nets["critic"])
        if disc is not None and "disc" in nets:
            _check_state_dict(path, "disc", disc, nets["disc"])
        for name, n in norms.items():
            if name in s["norms"]:
                _check_norm(path, name, n, s["norms"][name]["mean"])
        with torch.no_grad():
            for module, key in ((policy, "actor"), (critic, "critic"), (disc if disc is not None and "disc" in nets else None, "disc")):
                if module is not None:
                    for k, v in module.state_dict().items():
                        v.copy_(nets[key][k])
        if disc is not None and "disc" not in nets:
            _note(notes, "model file %s has no discriminator: the discriminator stays randomly initialised" % path)
        for name, n in norms.items():
            if name in s["norms"]:
                d = s["norms"][name]
                for fld in _NORM_FIELDS:
                    setattr(n, fld, d[fld].to(device=n.mean.device, dtype=torch.float32).clone())
                n.new_count = 0; n.new_sum.zero_(); n.new_sum_sq.zero_()
                counts[name] = int(d["count"])
    for name in norms:
        if name not in counts:
            _note(notes, "model file %s has no %s: it stays as initialised" % (path, name))
    return dict(kind=kind, counts=counts, notes=notes)
