"""Write a golden blob as several ``<stem>.<i>.npz`` files of at most ~900 KB each (tests/golden_util.load_shards reads
them back as one mapping), so that no committed fixture file is larger than 1 MB."""
import glob
import io
import os

import numpy as np

MAX_BYTES = 900_000


def save_shards(stem, blob):
    for old in glob.glob(stem + ".*.npz"):
        os.remove(old)
    shards, cur, size = [], {}, 0
    for k, v in blob.items():
        buf = io.BytesIO()
        np.savez_compressed(buf, v)
        n = buf.getbuffer().nbytes
        if cur and size + n > MAX_BYTES:
            shards.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += n
    shards.append(cur)
    for i, part in enumerate(shards):
        np.savez_compressed(f"{stem}.{i}.npz", **part)
    return [f"{stem}.{i}.npz" for i in range(len(shards))]
