"""The oracle's record of the reference's per-chain bookkeeping (restbits, excess_state_len, push depths) against the
reference-classes golden traces, and StreamSet.bit_accounting's arithmetic against cifar_compress.py:253-259 written out
literally.  CPU only."""

import numpy as np
import pytest
import torch

from codec_harness import bitswap_golden
from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200.config import preset
from bitswap_b200.streams import StreamSet

def _chain(name, scheme, nimg=None):
    """The golden run's inputs through the oracle (coder "c", torch-CPU pmfs) -> (record, trace, golden)."""
    g = bitswap_golden(name)
    cfg = preset(name)
    torch.set_num_threads(4)
    m = O.ModelOracle(cfg, synthetic.synthetic_state_dict(cfg, seed=50, varied=True))
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    trace, record = [], {}
    bs = O.BitSwapOracle(cfg, m, zend, zcen, coder="c", pmf="torch", trace=trace, record=record)
    imgs = synthetic.synthetic_images(cfg, g["nimg"], seed=7)
    w, head = synthetic.initial_words(g["nwords"], seed=100)
    st = O.CState(w, head)
    enc = bs.encode_image if scheme == "bitswap" else bs.encode_image_bbans
    for xi in range(nimg or g["nimg"]):
        st = enc(st, imgs[xi])
    return record, trace, g, st


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_bitswap_record_matches_reference_trace(name):
    """Bit-Swap: restbits is the state after the chain's first pop (cifar_compress.py:190-192) and excess_state_len the
    least length after any pop (demo_compress.py:137); both read off the reference-classes trace, which the oracle's own
    trace must equal entry for entry."""
    record, trace, g, _ = _chain(name, "bitswap")
    want = [tuple(e) for e in g["trace"][1:]]
    per = 2 * preset(name).nz + 1                                             # entries per image: nz pops, nz pushes, prior
    assert [(f"img{i // per} {t}", n, s) for i, (t, n, s) in enumerate(trace)] == want
    init_len = g["trace"][0][1]
    assert record["init_len"] == init_len == g["nwords"]
    assert record["rest_len"] == dict((t, n) for t, n, _ in want)["img0 pop z1"]
    assert record["excess_len"] == min([init_len] + [n for t, n, _ in want if " pop " in t])
    pushes = [(t.split(" ", 1)[1], n) for t, n, _ in want if " push " in t]
    assert record["push_lens"] == pushes and record["images"] == g["nimg"]
    assert max(n for _, n in record["push_lens"]) == g["final_len"]          # every push of this chain adds words


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_bbans_record_takes_restbits_after_the_last_pop(name):
    """BB-ANS: the reference takes restbits after all nz pops of the first image (cifar_compress.py:224-226), not after
    the first.  The trace has an entry after every pop and push; the record must agree with it, and with nz >= 2 the two
    rules give different lengths, which is what makes the rule observable."""
    cfg = preset(name)
    record, trace, g, st = _chain(name, "bbans")
    tags = [t for t, _, _ in trace]
    per_image = [f"pop z{i + 1}" for i in range(cfg.nz)] + ["push x"] + [f"push z{i}" for i in range(1, cfg.nz)] + ["push prior"]
    assert tags == per_image * g["nimg"]
    lens = [n for _, n, _ in trace]
    assert record["rest_len"] == lens[cfg.nz - 1]
    assert record["rest_len"] < lens[0]                                      # not the Bit-Swap rule: later pops took more
    assert record["excess_len"] == min([record["init_len"]] + [n for t, n, _ in trace if t.startswith("pop")])
    assert record["push_lens"] == [(t, n) for t, n, _ in trace if t.startswith("push")]
    assert lens[-1] == st.n + 1 and trace[-1][2] == st.digest()


def test_record_spans_the_chain_not_one_image():
    """restbits is taken once per chain: coding a second image leaves it where the first image put it, while the excess
    length and the push list keep growing with the chain."""
    r1, _, _, _ = _chain("tiny", "bitswap", nimg=1)
    r2, _, _, _ = _chain("tiny", "bitswap", nimg=2)
    assert r1["rest_len"] == r2["rest_len"] and r2["images"] == 2 and r1["images"] == 1
    assert r2["push_lens"][:len(r1["push_lens"])] == r1["push_lens"] and len(r2["push_lens"]) == 2 * len(r1["push_lens"])
    assert r2["excess_len"] <= r1["excess_len"]


def _reference_logging(init_len, rest_len, state_lens, xdim):
    """cifar_compress.py:252-259 as written, for one experiment whose state after image xi has length state_lens[xi]."""
    n = len(state_lens)
    nets, cma, total, added = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n)
    for xi in range(n):
        totaladdedbits = (state_lens[xi] - init_len) * 32
        totalbits = (state_lens[xi] - (rest_len - 1)) * 32
        nets[xi] = (totaladdedbits / xdim) - nets[:xi].sum()
        cma[xi] = totalbits / (xdim * (xi + 1))
        total[xi] = totalbits
        added[xi] = totaladdedbits
    return nets, cma, total, added


class _Sizes:
    """Stands in for a device StreamSet: bit_accounting reads only sizes() and rest_words()."""

    def __init__(self, nwords, rest):
        self.n_, self.rest_ = np.asarray(nwords, dtype=np.int64), np.asarray(rest, dtype=np.int64)

    def sizes(self):
        return self.n_, np.zeros(self.n_.size, np.uint64), np.zeros(self.n_.size, np.int32)

    def rest_words(self):
        return self.rest_


@pytest.mark.parametrize("name", ["tiny", "tiny3"])
def test_bit_accounting_is_the_reference_arithmetic(name):
    """Per image of the golden chain and of two made-up chains (one per stream), bit_accounting equals the reference's
    nets (as their running mean), cma, total and totaladdedbits."""
    g = bitswap_golden(name)
    cfg = preset(name)
    init = g["trace"][0][1]
    rest = dict((t, n) for t, n, _ in g["trace"])["img0 pop z1"]
    after = [n for t, n, _ in g["trace"] if t.endswith("push prior")]
    chains = [(init, rest, after), (3001, 2900, [3400, 3950, 4100]), (33, 2, [700, 1500, 2222])]
    for xi in range(len(after)):
        for i0, r0, lens in chains:
            got = StreamSet.bit_accounting(_Sizes([lens[xi] - 1], [r0 - 1]), i0 - 1, cfg.xdim, xi + 1)
            nets, cma, total, added = _reference_logging(i0, r0, lens[:xi + 1], cfg.xdim)
            assert got["cma_bits_per_dim"][0] == pytest.approx(cma[xi], rel=1e-15)
            assert got["total_bits"][0] == total[xi] and got["total_added_bits"][0] == added[xi]
            assert got["net_bits_per_dim"][0] == pytest.approx(nets[:xi + 1].mean(), rel=1e-12)
    # all chains at once: one CMA and one total per stream, each from that stream's own rest words
    xi = len(after) - 1
    got = StreamSet.bit_accounting(_Sizes([c[2][xi] - 1 for c in chains], [c[1] - 1 for c in chains]), init - 1, cfg.xdim,
                                   xi + 1)
    ref = [_reference_logging(i0, r0, lens, cfg.xdim) for i0, r0, lens in chains]
    assert np.allclose(got["cma_bits_per_dim"], [r[1][xi] for r in ref], rtol=1e-15, atol=0)
    assert np.array_equal(got["total_bits"], [r[2][xi] for r in ref])
    assert StreamSet.bit_accounting(_Sizes([after[-1] - 1], [rest - 1]), init - 1, cfg.xdim, g["nimg"])["net_bits_per_dim"][0] \
        == g["net_bits_per_dim"]
