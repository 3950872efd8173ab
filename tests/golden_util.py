"""Loader for tests/golden/inet_cases.*.npz (generated from the reference source by
oracle/gen_golden.py)."""
import ast
import glob
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "inet_cases")


class Shards:
    """The arrays of ``<stem>.<i>.npz`` (written by oracle/shards.py) as one mapping with an ``.files`` list."""

    def __init__(self, stem):
        paths = sorted(glob.glob(stem + ".*.npz"), key=lambda p: int(p.rsplit(".", 2)[1]))
        if not paths:
            raise FileNotFoundError(stem + ".*.npz")
        self._src = {}
        for path in paths:
            z = np.load(path, allow_pickle=False)
            for k in z.files:
                self._src[k] = z
        self.files = list(self._src)

    def __getitem__(self, k):
        return self._src[k][k]

    def __contains__(self, k):
        return k in self._src


def load_shards(stem):
    return Shards(stem)


class GoldenCase:
    """One case of tests/golden/inet_cases.*.npz (generated from the reference source
    by oracle/gen_golden.py)."""

    def __init__(self, blob, name):
        self.name = name
        pre = name + "/"
        meta = [str(x) for x in blob[pre + "meta"]]
        self.cls = meta[0]
        self.B = int(meta[1])
        self.same = bool(int(meta[2]))
        self.kwargs = ast.literal_eval(meta[3])
        self.t = {}
        self.params = {}
        self.gparams = {}
        for k in blob.files:
            if not k.startswith(pre) or k == pre + "meta":
                continue
            sub = k[len(pre):]
            v = torch.from_numpy(blob[k])
            if sub.startswith("param/"):
                self.params[sub[6:]] = v
            elif sub.startswith("gparam/"):
                self.gparams[sub[7:]] = v
            else:
                self.t[sub] = v

    @property
    def propagation(self):
        return self.cls == "PropagationNet"


def load_golden_cases():
    blob = load_shards(GOLDEN)
    return [GoldenCase(blob, str(n)) for n in blob["__names__"]]
