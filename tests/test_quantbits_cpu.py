"""quantbits 11 and 12 (2048 and 4096 bins per latent dimension) without a GPU: the oracle and the top-level bins against
a known-answer test the reference's own classes produced at S = 4096 (tests/golden/make_golden_q12.py), and the
argument checks that refuse quantbits 13 before any device work."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200.codec import Bins as DeviceBins, check_quantbits, MAX_QUANTBITS
from bitswap_b200.config import preset, with_
from bitswap_b200.rand import Bins

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KAT = json.load(open(os.path.join(GOLDEN, "ans_kat_q12.json")))[0]


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def kat_inputs():
    rs = np.random.RandomState(KAT["seed"])
    pm = rs.dirichlet(np.ones(KAT["S"]) * 0.5, size=KAT["L"])
    sym = rs.randint(0, KAT["S"], size=KAT["L"])
    w, head = synthetic.initial_words(KAT["N"], seed=100)
    return pm, sym, w, head


def test_kat_shape():
    assert (KAT["S"], KAT["q"]) == (4096, 12) and KAT["L"] >= 256


def test_kat_q12_tables_and_coder():
    pm, sym, w, head = kat_inputs()
    assert O.state_digest(w, head) == KAT["init_sha"]
    P, C = O.tables_c(pm, 31, 12)
    P2, C2 = O.tables_np(pm, 31, 12)
    assert np.array_equal(P, P2) and np.array_equal(C, C2)
    assert [int(v) for v in P[0, :6]] == KAT["P_row0_head"]
    assert _sha(P) == KAT["P_sha"] and _sha(C) == KAT["C_sha"]
    a = O.AnsC(tables=(P, C))
    st = a.encode(O.CState(w, head), sym)
    assert (st.n + 1, hex(st.head), st.digest()) == (KAT["push_len"], KAT["push_head"], KAT["push_sha"])
    st2, psym = a.decode(O.CState(w, head))
    assert (st2.n + 1, hex(st2.head), st2.digest()) == (KAT["pop_len"], KAT["pop_head"], KAT["pop_sha"])
    assert [int(v) for v in psym[:6]] == KAT["pop_syms_head"] and _sha(psym.astype(np.int64)) == KAT["pop_syms_sha"]
    st3, rsym = a.decode(st)                                  # both inverses
    assert np.array_equal(rsym, sym) and st3.digest() == KAT["init_sha"]
    assert a.encode(st2, psym).digest() == KAT["init_sha"]


def test_kat_q12_port_literal():
    pm, sym, w, head = kat_inputs()
    a = O.AnsPort(pm, 31, 12)
    init = [int(v) for v in w] + [head]
    pushed = a.encode(init.copy(), sym)
    assert (len(pushed), hex(pushed[-1])) == (KAT["push_len"], KAT["push_head"])
    assert O.CState.from_list(pushed).digest() == KAT["push_sha"]
    popped, ps = a.decode(init.copy())
    assert (len(popped), hex(popped[-1])) == (KAT["pop_len"], KAT["pop_head"])
    assert [int(v) for v in ps[:6]] == KAT["pop_syms_head"]


def test_top_level_bins_q12_match_reference():
    g = np.load(os.path.join(GOLDEN, "bins_q12.npz"))
    b = Bins(torch.zeros((1, 1, 3)), torch.ones((1, 1, 3)), 12)
    assert b.endpoints().dtype == torch.float32 and b.endpoints().shape == (1, 1, 3, 4095)
    assert np.array_equal(b.endpoints().numpy(), g["top_end"]) and np.array_equal(b.centres().numpy(), g["top_cen"])


@pytest.mark.parametrize("q", [0, 13, 16, 10.0])
def test_out_of_range_quantbits_are_refused_before_device_work(q):
    with pytest.raises(ValueError):
        check_quantbits(q)
    cfg = with_(preset("tiny"), quantbits=q)
    with pytest.raises(ValueError):       # raised before any CUDA call: this runs on machines without a GPU
        DeviceBins(cfg, np.zeros((2, 256, 1)), np.zeros((2, 256, 2)))


def test_supported_quantbits_pass_the_check():
    for q in range(1, MAX_QUANTBITS + 1):
        check_quantbits(q)
    assert with_(preset("cifar8"), quantbits=12).zsupport == 4096


def test_abi_bins_create_refuses_q13():
    """bsw_bins_create validates its arguments before allocating anything, so the C ABI answers without a GPU."""
    from bitswap_b200 import _lib
    _lib.build()
    L = _lib.lib()
    h = ctypes.c_void_p()
    one = np.zeros(8, dtype=np.float64)
    assert L.bsw_bins_create(ctypes.byref(h), 1, 1, 13, 1024, one.ctypes.data, one.ctypes.data) == 4
    assert b"bad arguments" in L.bsw_last_error() and not h.value
    assert L.bsw_bins_create(ctypes.byref(h), 1, 1, 0, 1024, one.ctypes.data, one.ctypes.data) == 4
