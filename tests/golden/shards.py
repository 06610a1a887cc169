"""Golden fixtures larger than a file should be are stored as shards: <name>.<i>.pt, each a dict {entry path: value} of at most
SHARD_BYTES serialized bytes, where an entry path is (key,) or (key, sub_key) for the members of a dict-valued entry (state dicts,
gradients).  load() puts the original nested dict back together."""
import glob
import io
import os

import torch

SHARD_BYTES = 900_000


def _nbytes(v):
    b = io.BytesIO()
    torch.save(v, b)
    return b.tell()


def save(obj, directory, name):
    for old in glob.glob(os.path.join(directory, name + ".*.pt")):
        os.remove(old)
    entries = []
    for k, v in obj.items():
        if isinstance(v, dict) and v:
            entries += [((k, sk), sv) for sk, sv in v.items()]
        else:
            entries.append(((k,), v))
    shards, cur, size = [], {}, 0
    for path, v in entries:
        n = _nbytes(v)
        if cur and size + n > SHARD_BYTES:
            shards.append(cur)
            cur, size = {}, 0
        cur[path] = v
        size += n
    shards.append(cur)
    for i, sh in enumerate(shards):
        torch.save(sh, os.path.join(directory, "%s.%d.pt" % (name, i)))


def load(directory, name):
    out = {}
    files = sorted(glob.glob(os.path.join(directory, name + ".*.pt")), key=lambda p: int(p.rsplit(".", 2)[1]))
    assert files, "no shards of %s in %s" % (name, directory)
    for f in files:
        for path, v in torch.load(f, weights_only=False).items():
            if len(path) == 1:
                out[path[0]] = v
            else:
                out.setdefault(path[0], {})[path[1]] = v
    return out
