"""Secondary measurement: e2e through `extract_batch` for the container types the reference's callers actually pass —
a LIST of numpy arrays (compute_and_store_features_batch, set.py:2384) and a list of CPU torch tensors (OnTheFlyFeatures,
input_strategies.py:441) — against the (B, n) array route that bench.py's e2e times.  Also the raw host-copy rates that
bound the list routes (pinned staging copy with 1..8 threads)."""
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import lhotse_b200 as lb

SR, B, n = 16000, 1024, 160000
hours = B * n / SR / 3600


def timeit(fn, reps=4):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    rs = np.random.RandomState(0)
    ext = lb.B200Fbank()
    arr = torch.empty((B, n), dtype=torch.float32, pin_memory=True).numpy()
    arr[:] = 0.1 * rs.randn(B, n).astype(np.float32)
    lst = [np.ascontiguousarray(arr[i]).copy() for i in range(B)]          # pageable, separately allocated (like decoder output)
    tl = [torch.from_numpy(a) for a in lst]
    import lhotse_b200.engine as E

    def legacy_numpy():  # what shipped before: one host thread gathers everything, then the C call
        keep = E.STAGING_THREADS
        E.STAGING_THREADS = 1
        try:
            buf, lens, offs = E.stage_host(lst)
            return ext.engine.extract_host(buf, lens, offsets=offs)
        finally:
            E.STAGING_THREADS = keep

    def legacy_torch():
        keep = E.STAGING_THREADS
        E.STAGING_THREADS = 1
        try:
            return ext.extract_batch_padded(tl, SR)
        finally:
            E.STAGING_THREADS = keep

    print(json.dumps({"staging_threads": E.STAGING_THREADS, "cpu_count": os.cpu_count()}), flush=True)
    pageable = arr.copy()
    eng = ext.engine
    for name, fn in (("(B, n) pinned array (bench.py e2e)", lambda: ext.extract_batch(arr, SR)),
                     ("(B, n) pageable array handed to the C call as is (before)", lambda: eng.extract_host(pageable.reshape(-1), [n] * B)),
                     ("(B, n) pageable array", lambda: ext.extract_batch(pageable, SR)),
                     ("list of numpy arrays, single-thread staging then C call (before)", legacy_numpy),
                     ("list of CPU torch tensors -> padded device tensor, single-thread staging (before)", legacy_torch),
                     ("list of numpy arrays (C-side gather: b200feat_extract_host_ptrs)", lambda: ext.extract_batch(lst, SR)),
                     ("list of CPU torch tensors -> device features", lambda: ext.extract_batch(tl, SR)),
                     ("list of CPU torch tensors -> padded device tensor", lambda: ext.extract_batch_padded(tl, SR))):
        t = timeit(fn)
        print(json.dumps({"route": name, "ms": t * 1e3, "h_per_s": hours / t}), flush=True)
    # raw staging copy: B arrays -> one pinned buffer
    stage = torch.empty(B * n, dtype=torch.float32, pin_memory=True)
    v = stage.numpy()
    for nt in (1, 2, 4, 8, 16):
        def cp(i):
            v[i * n:(i + 1) * n] = lst[i]
        with ThreadPoolExecutor(nt) as ex:
            list(ex.map(cp, range(B)))
            t0 = time.perf_counter()
            for _ in range(3):
                list(ex.map(cp, range(B)))
            t = (time.perf_counter() - t0) / 3
        print(json.dumps({"what": "staging copy into pinned memory", "threads": nt, "GBps": B * n * 4 / t / 1e9, "h_per_s": hours / t}), flush=True)


if __name__ == "__main__":
    main()
