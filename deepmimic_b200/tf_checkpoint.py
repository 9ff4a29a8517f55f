"""Minimal reader for TensorFlow-1 "TensorBundle" checkpoints (<prefix>.index + <prefix>.data-00000-of-00001), enough for the reference's
pretrained policies (R/data/policies/**.ckpt, written by tf.train.Saver in R/learning/tf_agent.py:60-66).  No TensorFlow needed.

The .index file is a LevelDB-format table (uncompressed blocks of prefix-compressed key/value entries, a block index and a 48-byte footer
with the magic 0xdb4775248b80fb57); each value is a BundleEntryProto {1: dtype, 2: shape{2: dim{1: size}}, 3: shard_id, 4: offset, 5: size,
6: crc32c}.  Float32 tensors, and the int32 sample counts of the normalisers, in a single data shard are read (that is what the reference
writes)."""
import os
import struct

import numpy as np

_MAGIC = 0xdb4775248b80fb57


def _varint(buf, pos):
    shift = result = 0
    while True:
        b = buf[pos]; pos += 1
        result |= (b & 0x7F) << shift
        if not (b & 0x80):
            return result, pos
        shift += 7


def _read_block(data, offset, size):
    block = data[offset:offset + size]
    if data[offset + size] != 0:
        raise ValueError("compressed checkpoint index blocks are not supported")
    n_restarts = struct.unpack_from("<I", block, len(block) - 4)[0]
    end = len(block) - 4 - 4 * n_restarts
    pos, key, out = 0, b"", []
    while pos < end:
        shared, pos = _varint(block, pos)
        non_shared, pos = _varint(block, pos)
        vlen, pos = _varint(block, pos)
        key = key[:shared] + block[pos:pos + non_shared]; pos += non_shared
        out.append((key, block[pos:pos + vlen])); pos += vlen
    return out


def _parse_entry(buf):
    """BundleEntryProto -> dict(dtype, shape, shard, offset, size)."""
    e = dict(dtype=0, shape=[], shard=0, offset=0, size=0)
    pos = 0
    while pos < len(buf):
        tag, pos = _varint(buf, pos)
        field, wt = tag >> 3, tag & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
            if field == 1: e["dtype"] = v
            elif field == 3: e["shard"] = v
            elif field == 4: e["offset"] = v
            elif field == 5: e["size"] = v
        elif wt == 2:
            ln, pos = _varint(buf, pos)
            sub = buf[pos:pos + ln]; pos += ln
            if field == 2:      # TensorShapeProto
                p = 0
                while p < len(sub):
                    t, p = _varint(sub, p)
                    if (t & 7) == 2:
                        l2, p = _varint(sub, p)
                        dim = sub[p:p + l2]; p += l2
                        if (t >> 3) == 2:
                            size, q = 0, 0
                            while q < len(dim):
                                t2, q = _varint(dim, q)
                                if (t2 & 7) == 0:
                                    v, q = _varint(dim, q)
                                    if (t2 >> 3) == 1: size = v
                                elif (t2 & 7) == 2:
                                    l3, q = _varint(dim, q); q += l3
                            e["shape"].append(size)
                    elif (t & 7) == 0:
                        _, p = _varint(sub, p)
        elif wt == 5:
            pos += 4
        elif wt == 1:
            pos += 8
        else:
            raise ValueError("unexpected protobuf wire type %d" % wt)
    return e


def list_entries(prefix):
    data = open(prefix + ".index", "rb").read()
    if struct.unpack_from("<Q", data, len(data) - 8)[0] != _MAGIC:
        raise ValueError("%s.index is not a TensorBundle index" % prefix)
    footer = data[-48:]
    pos = 0
    _, pos = _varint(footer, pos); _, pos = _varint(footer, pos)          # metaindex handle
    ioff, pos = _varint(footer, pos); isz, pos = _varint(footer, pos)      # index handle
    entries = {}
    for _, handle in _read_block(data, ioff, isz):
        boff, p = _varint(handle, 0); bsz, p = _varint(handle, p)
        for key, val in _read_block(data, boff, bsz):
            if key:                                                        # the empty key holds the BundleHeaderProto
                entries[key.decode()] = _parse_entry(val)
    return entries


_DTYPES = {1: "<f4", 3: "<i4"}   # TF DataType DT_FLOAT, DT_INT32


def load_checkpoint(prefix, int32=False):
    """All float32 tensors of the checkpoint as {name: ndarray}; with int32 the int32 tensors too (the normalisers' sample counts)."""
    entries = list_entries(prefix)
    raw = open(prefix + ".data-00000-of-00001", "rb").read()
    out = {}
    for name, e in entries.items():
        if e["shard"] != 0 or e["dtype"] not in ((1, 3) if int32 else (1,)):
            continue
        n = int(np.prod(e["shape"])) if e["shape"] else 1
        if e["size"] != 4 * n:
            raise ValueError("size mismatch for %s" % name)
        out[name] = np.frombuffer(raw, dtype=_DTYPES[e["dtype"]], count=n, offset=e["offset"]).reshape(e["shape"]).copy()
    return out


def load_actor(prefix):
    """The PPO actor of a reference checkpoint: hidden layers, mean head, log-std bias, and the state / action normalisers
    (R/learning/ppo_agent.py:52-90, tf_agent.py:101-131): <name>_mean, <name>_std and, when the checkpoint holds one, the int32 sample count
    <name>_count (agent/resource/<name>/count, a reading of the reference's normaliser that has not been checked against a checkpoint it
    wrote)."""
    t = load_checkpoint(prefix, int32=True)
    a = "agent/main/actor/"
    hidden = []
    k = 0
    while a + "%d/dense/kernel" % k in t:
        hidden.append((t[a + "%d/dense/kernel" % k], t[a + "%d/dense/bias" % k])); k += 1
    out = dict(hidden=hidden, mean=(t[a + "dist_gauss_diag/mean/kernel"], t[a + "dist_gauss_diag/mean/bias"]), logstd=t[a + "dist_gauss_diag/logstd/bias"])
    if a + "gate_common/0/dense/kernel" in t:
        # fc_2layers_gated_1024units (R/learning/nets/fc_2layers_gated_1024units.py): goal -> gate_common (128) -> per hidden layer a 64-unit
        # gate layer feeding a bias head (dense) and a scale head (dense_1)
        g = lambda name: (t[a + name + "/kernel"], t[a + name + "/bias"])
        out["gate_common"] = g("gate_common/0/dense")
        out["gates"] = [dict(hidden=g("gate%d/0/dense" % i), bias=g("gate%d/dense" % i), scale=g("gate%d/dense_1" % i)) for i in range(len(hidden))]
    _add_norms(out, t, ("s_norm", "g_norm", "a_norm"))
    return out


def load_critic(prefix):
    """The PPO critic of a reference checkpoint (PPOAgent._build_net_critic, R/learning/ppo_agent.py): the hidden layers under
    agent/main/critic/<i>/dense, the one-unit output layer agent/main/critic/dense, the gate layers of fc_2layers_gated_1024units named as in
    load_actor, and the value normaliser agent/resource/val_norm (plus s_norm / g_norm, which the critic shares with the actor) when present.
    These names follow the actor's scopes, and the normalisers' counts are read as load_actor reads them; neither has been checked against a
    checkpoint the reference wrote with its critic."""
    t = load_checkpoint(prefix, int32=True)
    c = "agent/main/critic/"
    g = lambda name: (t[c + name + "/kernel"], t[c + name + "/bias"])
    hidden = []
    while c + "%d/dense/kernel" % len(hidden) in t:
        hidden.append(g("%d/dense" % len(hidden)))
    out = dict(hidden=hidden, out=g("dense"))
    if c + "gate_common/0/dense/kernel" in t:
        out["gate_common"] = g("gate_common/0/dense")
        out["gates"] = [dict(hidden=g("gate%d/0/dense" % i), bias=g("gate%d/dense" % i), scale=g("gate%d/dense_1" % i)) for i in range(len(hidden))]
    _add_norms(out, t, ("s_norm", "g_norm", "val_norm"))
    return out


def _add_norms(out, t, names):
    for nm in names:
        for st in ("mean", "std", "count"):
            key = "agent/resource/%s/%s" % (nm, st)
            if key in t:
                out["%s_%s" % (nm, st)] = t[key]
