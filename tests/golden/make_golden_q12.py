"""Generates the quantbits-12 golden files by running the REFERENCE's own classes (same recipe as make_golden.py).

Run in the build container only (needs the reference checkout, read-only; BITSWAP_REFERENCE overrides its path):
    python tests/golden/make_golden_q12.py
The outputs are committed; nothing at test time reads the reference.

What is pinned:
  ans_kat_q12.json  KAT-4 of the reference `ANS` (cifar_compress.py:12-67) at S = 4096 bins, quantbits 12 -- the widest
                    support the device codec takes: tables, push, pop-first, both round trips
  bins_q12.npz      rand.Bins(0, 1, 12) top-level endpoints and centres (float32)
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import ANS, Bins, OUT, digest, init_state       # noqa: E402  (reference classes + shared helpers)


def ans_kat_q12():
    name, L, S, q, N, seed = "KAT-4", 256, 4096, 12, 4096, 4
    rs = np.random.RandomState(seed)
    pm = rs.dirichlet(np.ones(S) * 0.5, size=L)
    sym = rs.randint(0, S, size=L)
    a = ANS(torch.from_numpy(pm), 31, q)
    st0 = init_state(N)
    pushed = a.encode(st0.copy(), torch.from_numpy(sym))
    popped, psym = a.decode(st0.copy())
    rt1, rsym = a.decode(pushed.copy())
    rt2 = a.encode(popped.copy(), psym)
    assert rt1 == st0 and np.all(rsym.numpy() == sym) and rt2 == st0
    rec = dict(name=name, L=L, S=S, q=q, N=N, seed=seed, init_sha=digest(st0),
               push_len=len(pushed), push_head=hex(pushed[-1]), push_sha=digest(pushed),
               pop_len=len(popped), pop_head=hex(popped[-1]), pop_sha=digest(popped),
               pop_syms_sha=hashlib.sha256(psym.numpy().astype(np.int64).tobytes()).hexdigest()[:16],
               pop_syms_head=[int(v) for v in psym.numpy()[:6]],
               P_row0_head=[int(v) for v in a.pmfs[0, :6]],
               P_sha=hashlib.sha256(a.pmfs.astype(np.int64).tobytes()).hexdigest()[:16],
               C_sha=hashlib.sha256(a.cdfs.astype(np.int64).tobytes()).hexdigest()[:16])
    json.dump([rec], open(os.path.join(OUT, "ans_kat_q12.json"), "w"), indent=1)


def bins_q12():
    b = Bins(torch.zeros((1, 1, 3)), torch.ones((1, 1, 3)), 12)
    np.savez_compressed(os.path.join(OUT, "bins_q12.npz"), top_end=b.endpoints().numpy(), top_cen=b.centres().numpy())


if __name__ == "__main__":
    torch.set_num_threads(4)
    ans_kat_q12()
    bins_q12()
    print("quantbits-12 golden files written to", OUT)
