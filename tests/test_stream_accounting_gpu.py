"""Per-stream bookkeeping on the GPU: rest words, min words and bit_accounting against the reference's accounting as the
oracle records it; the packed (de)serialisation against a numpy restatement of the gather; and the word-stack capacity,
exact to the word, through every kind of push and through compress_images' retry loop."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from coder_harness import initial_states                               # noqa: E402
from codec_harness import gpu_oracle, setup                            # noqa: E402
from oracle import oracle as O                                         # noqa: E402
from bitswap_b200 import synthetic                                     # noqa: E402
from bitswap_b200.model import Model                                   # noqa: E402
from bitswap_b200.codec import BitSwapCodec, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.streams import StreamSet                             # noqa: E402
from bitswap_b200 import container                                     # noqa: E402

OVERFLOW = 2                                                           # BSW_E_OVERFLOW


def _reference_accounting(record, state_len, xdim, images):
    """cifar_compress.py:253-259 on the oracle's record of one chain."""
    totaladdedbits = (state_len - record["init_len"]) * 32
    totalbits = (state_len - (record["rest_len"] - 1)) * 32
    return dict(net_bits_per_dim=totaladdedbits / (xdim * images), cma_bits_per_dim=totalbits / (xdim * images),
                total_bits=totalbits, total_added_bits=totaladdedbits)


# ---------------------------------------------------------------------------------------------------------------------
# rest words, min words, bit_accounting
# ---------------------------------------------------------------------------------------------------------------------
PATHS = ["codec", "pipelined", "fused", "ext", "subrange"]


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name,scheme", [("tiny", BITSWAP), ("tiny", BBANS), ("tiny3", BITSWAP), ("tiny3", BBANS)])
def test_rest_min_words_and_accounting_vs_oracle(name, scheme, path):
    """Chains of 3 images on streams of distinct initial lengths.  After every image: each stream's state list, rest
    words (the reference's len(restbits) - 1: after the first pop for Bit-Swap, after the first image's nz pops for
    BB-ANS), min words (demo_compress.py's excess_state_len - 1) and every field of bit_accounting equal the oracle's
    record of the same chain.  Paths: BitSwapCodec; PipelinedCodec (2 lanes, overlap mode); the fused coder; the
    edge-coded _ext entry points with partial blocks; a sub-range call, which must leave the other streams alone."""
    B, nimg = 4, 3
    first, nstreams = (1, B + 2) if path == "subrange" else (0, B)
    cfg, m, sd, zend, zcen, bins, codec = setup(name, B)
    if path == "pipelined":
        codec = PipelinedCodec(cfg, sd, bins, B, lanes=2, use_tensor_cores=False)
        codec.set_dual_stream(True)
        net_model = codec.models[0]
    else:
        net_model = m
    if path == "fused":
        codec.set_two_phase(False)
    imgs = synthetic.synthetic_images(cfg, nimg * B, seed=61).reshape(nimg, B, *cfg.xs)
    exts = None
    if path == "ext":
        rs = np.random.RandomState(62)
        exts = rs.randint(1, 33, size=(nimg, B, 2)).astype(np.int16)
        exts[0, 0] = (32, 32)
        exts[1, 1] = (1, 1)
    states = initial_states(nstreams, seed=600, n=2500, step=37)
    ss = StreamSet(nstreams, 1 << 14)
    ss.import_lists(states)
    assert (ss.rest_words() == -1).all()
    records = [{} for _ in range(B)]
    orcs = [gpu_oracle(cfg, net_model, sd, zend, zcen, record=r) for r in records]
    ost = [O.CState.from_list(states[first + b]) for b in range(B)]
    enc = "encode_image" if scheme == BITSWAP else "encode_image_bbans"
    for xi in range(nimg):
        ext = None if exts is None else torch.from_numpy(exts[xi]).cuda()
        codec.encode(ss, torch.from_numpy(imgs[xi]).cuda(), first=first, scheme=scheme, extent=ext)
        torch.cuda.synchronize()
        ss.raise_on_error()
        for b in range(B):
            ost[b] = getattr(orcs[b], enc)(ost[b], imgs[xi, b], extent=None if exts is None else tuple(exts[xi, b]))
        got = ss.export_lists()
        n, _, _ = ss.sizes()
        rest, low = ss.rest_words(), ss.min_words()
        for b in range(B):
            s, r = first + b, records[b]
            acct = ss.bit_accounting(r["init_len"] - 1, cfg.xdim, xi + 1)
            want = _reference_accounting(r, len(ost[b].to_list()), cfg.xdim, xi + 1)
            if b == 0:
                print(f"{name} {'Bit-Swap' if scheme == BITSWAP else 'BB-ANS'} {path}: CMA@{xi + 1} "
                      f"{acct['cma_bits_per_dim'][s]:.4f} (reference {want['cma_bits_per_dim']:.4f}) bits/dim")
            assert got[s] == ost[b].to_list(), f"image {xi} stream {s}: state differs from the oracle"
            assert n[s] + 1 == len(got[s])
            assert rest[s] == r["rest_len"] - 1, f"image {xi} stream {s}: rest words {rest[s]}, reference {r['rest_len'] - 1}"
            assert low[s] == r["excess_len"] - 1, f"image {xi} stream {s}: min words {low[s]}, reference {r['excess_len'] - 1}"
            for k, v in want.items():
                assert acct[k][s] == v, f"image {xi} stream {s}: {k} {acct[k][s]} != reference {v}"
        for s in set(range(nstreams)) - set(range(first, first + B)):
            assert got[s] == states[s] and rest[s] == -1 and low[s] == len(states[s]) - 1


def test_fill_import_and_unpack_start_a_new_chain():
    """rest words go back to -1 wherever a new chain starts -- fill, import_lists, the plain and the trimmed unpack -- so
    that the next encode records the new chain's restbits instead of keeping the old chain's."""
    B = 3
    cfg, m, sd, zend, zcen, bins, codec = setup("tiny", B)
    imgs = torch.from_numpy(synthetic.synthetic_images(cfg, B, seed=63)).cuda()
    w, head = synthetic.initial_words(2000, seed=100)
    ss = StreamSet(B, 1 << 13)

    def coded():
        codec.encode(ss, imgs)
        torch.cuda.synchronize()
        ss.raise_on_error()
        r = ss.rest_words()
        assert (r > 0).all() and (r < 2000).all()
        return r

    ss.fill(w, head)
    assert (ss.rest_words() == -1).all()
    r0 = coded()
    ss.fill(w, head)
    assert (ss.rest_words() == -1).all()
    assert np.array_equal(coded(), r0)                    # the same chain again: the same restbits
    ss.import_lists(initial_states(B, seed=7, n=1500, step=37))
    assert (ss.rest_words() == -1).all()
    coded()
    words, offs, heads = (a.copy() for a in ss.export_packed())
    coded()                                               # rest words of a chain that the unpack must forget
    ss.import_packed_fast(words, offs, heads)
    torch.cuda.synchronize()
    assert (ss.rest_words() == -1).all() and (ss.sizes()[2] == 0).all()
    coded()
    words, offs, heads, base = (a.copy() for a in ss.export_packed(trim=True))
    ss.fill(w, head)
    coded()
    ss.fill(w, head)
    coded()
    ss.import_packed_fast(words, offs, heads, base=base)
    torch.cuda.synchronize()
    assert (ss.rest_words() == -1).all() and (ss.sizes()[2] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# packed serialisation
# ---------------------------------------------------------------------------------------------------------------------
CAP = 64


def _stream_set_with(n, lo, seed_words, seed_head, rows_above, heads):
    """A set whose stream b holds seed_words[:lo[b]] + rows_above[b] (n[b] words in all), min words lo[b], head heads[b]:
    made with fill + a trimmed unpack, then read back through the per-stream host paths (sizes, min_words, export),
    which do not use the pack kernels."""
    B = len(n)
    ss = StreamSet(B, CAP)
    assert ss.capacity == CAP
    ss.fill(seed_words, seed_head)
    offs = np.zeros(B + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows_above], out=offs[1:])
    flat = np.concatenate([np.asarray(r, dtype=np.uint32) for r in rows_above] + [np.zeros(1, np.uint32)])
    ss.unpack_device(torch.from_numpy(flat.view(np.int32)).cuda(), torch.from_numpy(offs).cuda(),
                     torch.from_numpy(np.asarray(heads, dtype=np.uint64).view(np.int64)).cuda(),
                     torch.from_numpy(np.asarray(lo, dtype=np.int32)).cuda())
    torch.cuda.synchronize()
    nn, hh, ff = ss.sizes()
    assert np.array_equal(nn, n) and np.array_equal(ss.min_words(), lo) and (ff == 0).all()
    assert np.array_equal(hh, np.asarray(heads, dtype=np.uint64))
    return ss


def _random_streams(B, seed):
    """Per-stream (n, lo, rows) covering zero-length streams, min words == n (nothing to send), n == capacity and
    ordinary ones, in a shuffled order."""
    rs = np.random.RandomState(seed)
    kind = rs.randint(0, 4, size=B)
    n = np.where(kind == 0, 0, np.where(kind == 2, CAP, rs.randint(1, CAP + 1, size=B))).astype(np.int64)
    lo = np.where(kind == 1, n, (rs.random_sample(B) * (n + 1)).astype(np.int64).clip(0, n)).astype(np.int64)
    kind[0], n[0], lo[0] = 2, CAP, 0                                 # a full stream, sent whole
    seed_words = rs.randint(0, 1 << 32, size=CAP, dtype=np.uint64).astype(np.uint32)
    rows = [rs.randint(0, 1 << 32, size=int(n[b] - lo[b]), dtype=np.uint64).astype(np.uint32) for b in range(B)]
    heads = rs.randint(1 << 32, 1 << 63, size=B, dtype=np.uint64)
    return n, lo, seed_words, rows, heads


def _np_pack(full_rows, n, lo, heads, first, count, trim):
    """The gather restated: offsets = exclusive prefix sum of the words sent, words = those words back to back."""
    sl = slice(first, first + count)
    base = np.minimum(lo[sl], n[sl]) if trim else np.zeros(count, dtype=np.int64)
    offs = np.zeros(count + 1, dtype=np.int64)
    np.cumsum(n[sl] - base, out=offs[1:])
    words = np.concatenate([full_rows[first + i][int(base[i]):int(n[first + i])] for i in range(count)]
                           + [np.zeros(0, np.uint32)]).astype(np.uint32)
    return words, offs, heads[sl], base


@pytest.mark.parametrize("count,first", [(1, 0), (1, 3), (1023, 0), (1024, 0), (1025, 0), (1025, 2), (2500, 1), (4100, 0),
                                         (4100, 5)])
@pytest.mark.parametrize("trim", [False, True])
def test_pack_unpack_vs_numpy(count, first, trim):
    """pack / pack_trimmed of streams [first, first + count) == the numpy gather: offsets, words, heads, bases.  The
    prefix sum of k_pack_offsets runs in rounds of 1024 streams with a carry between them; counts 1023 to 4100 cover
    one to five rounds.  Then the packed streams go back into a fresh set (for the trimmed form, one already holding the
    seed words): states, min words, flags and rest words must be those of the source."""
    B = first + count + 2                                            # streams on both sides of the range
    n, lo, seed_words, rows, heads = _random_streams(B, seed=count + 17 * first)
    full_rows = [np.concatenate([seed_words[:lo[b]], rows[b]]).astype(np.uint32) for b in range(B)]
    ss = _stream_set_with(n, lo, seed_words, 5, rows, heads)
    want_w, want_o, want_h, want_base = _np_pack(full_rows, n, lo, heads, first, count, trim)
    wd, od, hd, bd = ss.pack_device(first, count, trim=trim)
    torch.cuda.synchronize()
    o = od.cpu().numpy()
    assert np.array_equal(o, want_o), f"offsets differ first at {int(np.argmax(o != want_o))}"
    total = int(want_o[-1])
    assert np.array_equal(wd[:total].cpu().numpy().view(np.uint32), want_w)
    assert np.array_equal(hd.cpu().numpy().view(np.uint64), want_h)
    if trim:
        assert np.array_equal(bd.cpu().numpy(), want_base)
    # the host form is the same gather
    host = ss.export_packed(first, count, trim=trim)
    assert np.array_equal(host[0], want_w) and np.array_equal(host[1], want_o) and np.array_equal(host[2], want_h)
    host = tuple(a.copy() for a in host)
    fresh = StreamSet(B, CAP)
    if trim:
        fresh.fill(seed_words, 5)
    fresh.import_packed_fast(*host[:3], first=first, base=host[3] if trim else None)
    torch.cuda.synchronize()
    got = fresh.export_lists(first, count)
    for i in range(count):
        assert got[i] == [int(v) for v in full_rows[first + i]] + [int(heads[first + i])], f"stream {first + i}"
    fn, _, ff = fresh.sizes()
    assert np.array_equal(fn[first:first + count], n[first:first + count]) and (ff == 0).all()
    assert np.array_equal(fresh.min_words()[first:first + count], want_base if trim else n[first:first + count])
    assert (fresh.rest_words() == -1).all()


@pytest.mark.parametrize("trim", [False, True])
def test_unpack_flags_a_corrupt_length_and_leaves_its_neighbours_alone(trim):
    """A packed length that does not fit (lo + n > capacity) in the middle of the set: that stream is flagged
    BSW_E_OVERFLOW and keeps what it held, its neighbours are unpacked exactly.  (It is never the last stream, so even a
    guard that let one word through would write inside the allocation: into its neighbour's first word.)"""
    B, bad = 7, 3
    rs = np.random.RandomState(9)
    seed_words = rs.randint(0, 1 << 32, size=CAP, dtype=np.uint64).astype(np.uint32)
    lo = np.array([0, 5, 0, 10, 0, 1, 0], dtype=np.int32) if trim else np.zeros(B, dtype=np.int32)
    n_sent = np.array([20, 7, CAP, CAP - 9, 3, CAP - 1, 0], dtype=np.int64)
    if not trim:
        n_sent[bad] = CAP + 1
    assert lo[bad] + n_sent[bad] == CAP + 1
    rows = [rs.randint(0, 1 << 32, size=int(k), dtype=np.uint64).astype(np.uint32) for k in n_sent]
    heads = rs.randint(1 << 32, 1 << 63, size=B, dtype=np.uint64)
    ss = StreamSet(B, CAP)
    ss.fill(seed_words, 11)
    before = ss.export_lists()
    offs = np.zeros(B + 1, dtype=np.int64)
    np.cumsum(n_sent, out=offs[1:])
    flat = np.concatenate(rows).astype(np.uint32)
    ss.unpack_device(torch.from_numpy(flat.view(np.int32)).cuda(), torch.from_numpy(offs).cuda(),
                     torch.from_numpy(heads.view(np.int64)).cuda(), torch.from_numpy(lo).cuda() if trim else None)
    torch.cuda.synchronize()
    n, h, f = ss.sizes()
    got = ss.export_lists()
    assert f[bad] == OVERFLOW and got[bad] == before[bad]
    for b in set(range(B)) - {bad}:
        assert f[b] == 0
        want = ([int(v) for v in seed_words[:lo[b]]] if trim else []) + [int(v) for v in rows[b]] + [int(heads[b])]
        assert got[b] == want, f"stream {b}"
    with pytest.raises(OverflowError):
        ss.raise_on_error()
    # the host path refuses the same input before any device work; it holds every stream to its own base + length
    with pytest.raises(OverflowError):
        ss.import_packed_fast(flat, offs, heads, base=lo if trim else None)
    keep = np.array([b != bad for b in range(B)])
    offs_ok = np.zeros(int(keep.sum()) + 1, dtype=np.int64)
    np.cumsum(n_sent[keep], out=offs_ok[1:])
    ss.import_packed_fast(np.concatenate([rows[b] for b in range(B) if b != bad]).astype(np.uint32), offs_ok, heads[keep],
                          base=lo[keep] if trim else None)
    torch.cuda.synchronize()
    assert (ss.sizes()[2] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# capacity, exact to the word
# ---------------------------------------------------------------------------------------------------------------------
def _kind(tag):
    return "x" if tag == "push x" else "prior" if tag == "push prior" else "z"


@pytest.mark.parametrize("name,scheme,two_phase", [("tiny3", BBANS, True), ("tiny3", BBANS, False),
                                                   ("tiny", BITSWAP, True), ("tiny3", BITSWAP, False)])
def test_capacity_is_exact_to_the_word(name, scheme, two_phase):
    """Every stream holds the same chain state on top of its own number of bottom pad words, which are never popped, so
    its lengths are the oracle's plus its pad.  Pads put the chain's peak depth at capacity - 1, capacity and
    capacity + 1, and put the first length over capacity on each push that sets a new maximum (pixel, latent and prior
    pushes).  A stream is flagged BSW_E_OVERFLOW exactly when pad + peak > capacity, and every other stream -- each
    flagged one is followed by one that is not -- is bit-identical to the same run with ample capacity."""
    nimg = 2
    cfg, m, sd, zend, zcen, bins, _ = setup(name, 1)
    imgs = synthetic.synthetic_images(cfg, nimg, seed=65)
    w0, head0 = synthetic.initial_words(800, seed=101)
    record = {}
    orc = gpu_oracle(cfg, m, sd, zend, zcen, record=record)
    st = O.CState(w0, head0)
    for xi in range(nimg):
        st = (orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans)(st, imgs[xi])
    assert record["excess_len"] > 1                                 # the chain never reaches the pads
    pushes = [(t, n - 1) for t, n in record["push_lens"]]            # word counts after every push
    peak = max(n for _, n in pushes)
    cap = (peak + 40 + 31) // 32 * 32
    new_max, run = [], w0.size
    for t, n in pushes:
        if n > run:
            new_max.append((t, run, n))
            run = n
    kinds = {_kind(t) for t, _, _ in new_max}
    assert {"x", "prior"} <= kinds and (scheme == BITSWAP or "z" in kinds), new_max
    pads = [cap - peak - 1, cap - peak, cap - peak + 1] + [cap - n + 1 for _, _, n in new_max]
    pads = [p for p in pads if 0 <= p and p + w0.size <= cap]
    layout = []
    for p in pads:                                                  # each padded stream, then one with no pad
        layout += [p, 0]
    B = len(layout)
    rs = np.random.RandomState(66)
    states = [[int(v) for v in rs.randint(0, 1 << 32, size=p, dtype=np.uint64)] + [int(v) for v in w0] + [head0]
              for p in layout]
    m_b = Model.from_config(cfg, max_batch=B).load_state_dict(sd)
    m_b.compress()
    codec = BitSwapCodec(cfg, m_b, bins, B)
    codec.set_two_phase(two_phase)
    x = torch.from_numpy(np.ascontiguousarray(imgs)).cuda()
    res = {}
    big = cap + (max(layout) + 63) // 32 * 32
    for c in (cap, big):
        ss = StreamSet(B, c)
        assert ss.capacity == c
        ss.import_lists(states)
        for xi in range(nimg):
            codec.encode(ss, x[xi:xi + 1].expand(B, *cfg.xs).contiguous(), scheme=scheme)
        torch.cuda.synchronize()
        res[c] = (ss.export_lists(), ss.sizes()[2])
    ample, f_ample = res[big]
    assert (f_ample == 0).all()
    want = st.to_list()
    for b, p in enumerate(layout):
        assert ample[b] == states[b][:p] + want, f"stream {b} (pad {p}) differs from the oracle"
    tight, f = res[cap]
    expect = np.array([OVERFLOW if p + peak > cap else 0 for p in layout], dtype=np.int32)
    assert np.array_equal(f, expect), list(zip(layout, f.tolist(), expect.tolist()))
    for b in np.nonzero(expect == 0)[0]:
        assert tight[b] == ample[b], f"stream {b} (pad {layout[b]}) differs from the ample run"
    print(f"{name} scheme {scheme} two_phase {two_phase}: capacity {cap}, peak {peak}, new maxima "
          f"{[(t, n) for t, _, n in new_max]}, {int((expect != 0).sum())} of {B} streams flagged")


def _push_level(entry, ss, B, L, S, q, mu, sc, ends, sym):
    """One level of L symbols pushed onto streams [0, B) through one push entry point of the C ABI."""
    from bitswap_b200._lib import lib, check, cuda_stream_ptr
    dmu = torch.from_numpy(np.tile(mu, (B, 1))).cuda()
    dsc = torch.from_numpy(np.tile(sc, (B, 1))).cuda()
    e_pad = np.full((L, S), 1e300)
    e_pad[:, :S - 1] = ends
    de = torch.from_numpy(e_pad).cuda()
    s16 = torch.from_numpy(np.tile(sym.astype(np.int16), (B, 1))).cuda()
    if entry == "k_push_pairs":
        nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        check(lib().bsw_logistic_push_2p(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, de.data_ptr(), S,
                                         s16.data_ptr(), L, S, 31, q, scratch.data_ptr(), nbytes, cuda_stream_ptr()))
    elif entry == "k_logistic_push":
        check(lib().bsw_logistic_push(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, de.data_ptr(), S,
                                      s16.data_ptr(), L, S, 31, q, cuda_stream_ptr()))
    else:
        pm = O.logistic_pmfs_torch(torch.from_numpy(ends).cuda(), torch.from_numpy(mu.astype(np.float64)).cuda(),
                                   torch.from_numpy(sc.astype(np.float64)).cuda()).cpu().numpy()
        P, C = O.tables_c(pm, 31, q)
        dP = torch.from_numpy(P.astype(np.uint32).view(np.int32)).cuda()
        dC = torch.from_numpy(C.astype(np.uint32).view(np.int32)).cuda()
        s32 = torch.from_numpy(np.tile(sym.astype(np.int32), (B, 1))).cuda()
        check(lib().bsw_ans_push(ss.handle, 0, B, dP.data_ptr(), dC.data_ptr(), 0, 0, s32.data_ptr(), L, S, 31,
                                 cuda_stream_ptr()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("entry", ["k_push_pairs", "k_logistic_push", "k_push_tables"])
def test_each_push_kernel_fills_its_stream_to_the_last_word(entry):
    """Each push kernel on its own: one level pushed onto streams whose pads put the final depth at capacity - 1,
    capacity and capacity + 1.  Only the last is flagged; the other two, and the unpadded stream after each, are
    bit-identical to the same push with ample capacity.  (The codec's chains end on the prior push, so only this test
    lets a pixel or latent push end exactly at capacity.)"""
    L, S, q = 700, 64, 6
    rs = np.random.RandomState(68)
    ends = np.sort(rs.uniform(-6, 6, (L, S - 1)), axis=1)
    mu = rs.uniform(-2, 2, L).astype(np.float32)
    sc = rs.uniform(0.1, 1.5, L).astype(np.float32)
    sym = rs.randint(0, S, L)
    w0, head0 = synthetic.initial_words(100, seed=102)
    base = [int(v) for v in w0] + [head0]
    probe = StreamSet(1, 4096)
    probe.import_lists([base])
    _push_level(entry, probe, 1, L, S, q, mu, sc, ends, sym)
    probe.raise_on_error()
    peak = int(probe.sizes()[0][0])
    assert peak > len(base) + 32                                     # the level pushes whole windows of words
    cap = (peak + 40 + 31) // 32 * 32
    layout = [cap - peak - 1, 0, cap - peak, 0, cap - peak + 1, 0]
    states = [[int(v) for v in rs.randint(0, 1 << 32, size=p, dtype=np.uint64)] + base for p in layout]
    res = {}
    for c in (cap, cap + 1024):
        ss = StreamSet(len(layout), c)
        ss.import_lists(states)
        _push_level(entry, ss, len(layout), L, S, q, mu, sc, ends, sym)
        res[c] = (ss.export_lists(), ss.sizes()[2])
    ample, f_ample = res[cap + 1024]
    assert (f_ample == 0).all() and ample[1] == probe.export_lists()[0]
    tight, f = res[cap]
    assert f.tolist() == [0, 0, 0, 0, OVERFLOW, 0]
    for b in (0, 1, 2, 3, 5):
        assert tight[b] == ample[b], f"stream {b} (pad {layout[b]})"
    assert len(tight[2]) - 1 == cap                                 # the stream that ends exactly full


def test_compress_images_retries_until_the_chains_fit():
    """compress_images starts every chain with words_per_block words per block of room and doubles it after an overflow
    (four attempts).  With too little room for the first attempts the containers equal those of an ample run; with too
    little room for every attempt OverflowError is raised."""
    name = "tiny"
    cfg, m, sd, zend, zcen, bins, codec = setup(name, 3)
    rs = np.random.RandomState(67)
    images = [rs.randint(0, 256, (h, w, 1)).astype(np.uint8) for h, w in [(64, 64), (32, 96), (32, 32)]]
    made = []

    class Counting(StreamSet):
        def __init__(self, n, cap, device=None):
            made.append(cap)
            super().__init__(n, cap, device=device)
    real = container.StreamSet
    container.StreamSet = Counting
    try:
        ample = container.compress_images(codec, images, excess_state_len=1000, words_per_block=4000)
        assert len(made) == 1
        made.clear()
        tight = container.compress_images(codec, images, excess_state_len=1000, words_per_block=100)
        attempts = len(made)
        made.clear()
        with pytest.raises(OverflowError):
            container.compress_images(codec, images, excess_state_len=1000, words_per_block=1)
        assert len(made) == 4
    finally:
        container.StreamSet = real
    print(f"words_per_block 100: {attempts} attempts")
    assert attempts >= 2
    assert all(np.array_equal(a, b) for a, b in zip(ample, tight))
