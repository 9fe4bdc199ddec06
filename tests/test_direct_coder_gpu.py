"""The direct-cdf coder on the GPU.

(a) bsw_direct_tables equals the quantiser (direct_harness.direct_tables) applied to torch-CUDA's float64 sigmoid, bit for
    bit, at every support from 32 to 4096 bins, on the pixel row with row stride 0, on hostile rows and grid families 2-4.
(b) bsw_direct_pop / bsw_direct_push equal the numpy reference coder on those tables: symbols, heads, word counts and word
    stacks, from heads exactly on the bin edges and the renormalisation points, and on whole multi-row levels.
(c) The codec with coder="direct" equals the oracle recursion driven by the same GPU nets with direct tables, for Bit-Swap
    and BB-ANS, in split and bf16 arithmetic; overlap mode, lane splits, containers, regions and archives; an archive
    decoded with the other coder fails its initial-state check; and the refusals."""
import numpy as np
import pytest
import torch

import coder_harness as H
from codec_harness import gpu_oracle
from direct_harness import DirectOracle, direct_level, direct_tables, torch_cdfs
from oracle import oracle as O
from bitswap_b200 import synthetic
from bitswap_b200._lib import BswError, check, cuda_stream_ptr, lib
from bitswap_b200.codec import BBANS, BITSWAP, Bins, BitSwapCodec, PipelinedCodec
from bitswap_b200.config import preset, with_
from bitswap_b200.container import (compress_archive, compress_images, decompress_archive, decompress_images,
                                    decompress_regions)
from bitswap_b200.model import Model
from bitswap_b200.streams import StreamSet

pytestmark = pytest.mark.gpu

SUPPORTS = [32, 64, 128, 256, 512, 1024, 2048, 4096]
PIXEL_ROW = ((np.arange(1, 256) - 127.5) / 127.5) - 1.0 / 255.0        # ImageBins endpoints (rand.py:146-147)


def special_rows(S, rs, L=48):
    """Endpoint rows [L, S - 1] and float32 mu, sigma [L]: ordinary, needle, every bin live, mu beyond either end and on an
    edge, constant rows, runs of equal endpoints, NaN mu and NaN sigma."""
    lo, hi = -6 - rs.uniform(0, 1, L), 6 + rs.uniform(0, 1, L)
    ends = H.linspace_rows(lo, hi, S)
    mu = rs.normal(0, 1.5, L).astype(np.float32)
    sc = rs.uniform(0.1, 1.0, L).astype(np.float32)
    sc[0::8] = np.float32(1e-6)                                            # needle
    sc[1::8] = rs.uniform(20, 60, sc[1::8].shape)                          # every bin live
    mu[2::8] = rs.choice([-40.0, 40.0], mu[2::8].shape)                    # beyond either end
    mu[3::8] = ends[3::8, S // 3]                                          # on an edge
    ends[4::8] = rs.normal(0, 1, (ends[4::8].shape[0], 1))                 # constant rows
    runs = np.sort(np.repeat(rs.normal(0, 1, (ends[5::8].shape[0], S // 4)), 4, axis=1)[:, :S - 1], axis=1)
    ends[5::8] = runs                                                      # runs of equal endpoints
    mu[6] = np.float32("nan")
    sc[7] = np.float32("nan")
    return ends, mu, sc.astype(np.float32)


def device_tables(ends, mu, sc, S, ers=None):
    """bsw_direct_tables of rows ends ([L, S - 1], or one row with ers = 0) at float32 mu, sc [L] up-cast to double."""
    L = mu.size
    e = torch.from_numpy(np.ascontiguousarray(ends, dtype=np.float64)).cuda()
    m = torch.from_numpy(mu.astype(np.float64)).cuda()
    s = torch.from_numpy(sc.astype(np.float64)).cuda()
    P = torch.empty((L, S), dtype=torch.int32, device="cuda")
    C = torch.empty((L, S + 1), dtype=torch.int32, device="cuda")
    check(lib().bsw_direct_tables(e.data_ptr(), S - 1 if ers is None else ers, m.data_ptr(), s.data_ptr(), 1, L, S, 31, 0,
                                  P.data_ptr(), C.data_ptr(), cuda_stream_ptr()))
    torch.cuda.synchronize()
    u = lambda t: t.cpu().numpy().view(np.uint32).astype(np.int64)       # noqa: E731
    return u(P), u(C)


def cases(S, seed):
    """(label, ends [L, S - 1], mu [L], sigma [L], shared row?) for support S."""
    rs = np.random.RandomState(seed)
    out = [("special", *special_rows(S, rs), False)]
    for fam in (2, 3, 4):
        ends, mu, sc = H.family_case(fam, 24, S, 1, seed + fam)
        out.append((f"family {fam}", ends, mu[0], sc[0], False))
    if S == 256:
        L = 96
        mu = rs.uniform(-1.1, 1.1, L).astype(np.float32)
        sc = np.exp(rs.uniform(np.log(1e-4), np.log(0.5), L)).astype(np.float32)
        out.append(("pixel row", np.broadcast_to(PIXEL_ROW, (L, 255)), mu, sc, True))
    return out


@pytest.mark.parametrize("S", SUPPORTS)
def test_tables_equal_the_formula_on_torch_sigmoid(S):
    for label, ends, mu, sc, shared in cases(S, S):
        P, C = device_tables(PIXEL_ROW if shared else ends, mu, sc, S, ers=0 if shared else None)
        wP, wC = direct_tables(torch_cdfs(ends, mu, sc))
        bad = np.flatnonzero((C != wC).any(axis=1))
        assert bad.size == 0, f"S={S} {label}: rows {bad[:6].tolist()} differ from the formula"
        assert np.array_equal(P, wP)
        assert (P >= 1).all() and (C[:, S] == 1 << 31).all()


def _states(heads, rs, nwords=40):
    return [[int(v) for v in rs.randint(0, 1 << 32, nwords, dtype=np.int64)] + [int(h)] for h in heads]


@pytest.mark.parametrize("S", SUPPORTS)
def test_pop_and_push_at_bin_edges_and_thresholds(S):
    """One-row levels with one shared endpoint row (row stride 0), one stream per (mu/sigma, symbol, head kind): the head
    sits on a bin's lower or upper edge, makes the decoded value 2^32 - 1 or 2^32, or sits at a push threshold.  Every
    endpoint row kind of the case is the shared row once; the streams take the mu/sigma of the rows of the same kind."""
    rs = np.random.RandomState(S + 11)
    for label, ends, mu, sc, shared in cases(S, S + 5):
        L = mu.size
        for k in ([0] if shared else range(8 if label == "special" else 4)):
            r = np.arange(k, L, 8) if label == "special" else np.arange(L)
            row = ends[k]
            tab = H.RowTables(*direct_tables(torch_cdfs(np.broadcast_to(row, (r.size, S - 1)), mu[r], sc[r])))
            pad = np.append(row, 1e300)[None]
            for pop, kinds in ((True, H.POP_KINDS), (False, H.PUSH_KINDS)):
                n = 48
                j = rs.randint(0, r.size, n * len(kinds))
                s = np.where(rs.random_sample(j.size) < 0.3, rs.choice([0, 1, S - 2, S - 1], j.size), rs.randint(0, S, j.size))
                x = np.empty(j.size, dtype=np.uint64)
                ok = np.empty(j.size, dtype=bool)
                for t, kind in enumerate(kinds):
                    sl = slice(t * n, (t + 1) * n)
                    x[sl], ok[sl] = (H.pop_heads(tab.P[j[sl], s[sl]], tab.C[j[sl], s[sl]], kind, rs) if pop
                                     else H.push_heads(tab.P[j[sl], s[sl]], kind, rs))
                j, s, x = j[ok], s[ok], x[ok]
                states = _states(x, rs)
                want = H.Stacks.from_lists(states, cap=256)
                m_, s_ = mu[r][j][:, None], sc[r][j][:, None]
                what = f"S={S} {label} row {k} {'pop' if pop else 'push'}"
                if pop:
                    ss, got = direct_level(True, pad, m_, s_, S, states, ers=0, cap=256)
                    H.assert_same(what, got, ss.export(), H.pop(tab, j[:, None], want), want)
                else:
                    ss, _ = direct_level(False, pad, m_, s_, S, states, sym=s[:, None], ers=0, cap=256)
                    H.push(tab, j[:, None], want, s[:, None])
                    H.assert_same(what, None, ss.export(), None, want)
                ss.raise_on_error()


@pytest.mark.parametrize("S", SUPPORTS)
def test_pop_then_push_whole_levels(S):
    """Multi-row levels of every case from seeded states: pop, then push other symbols, against the numpy coder."""
    B = 8
    for label, ends, mu1, sc1, shared in cases(S, S + 9):
        L = mu1.size
        rs = np.random.RandomState(L + S)
        mu = np.stack([mu1] + [np.roll(mu1, b) for b in range(1, B)]).astype(np.float32)
        sc = np.stack([sc1] + [np.roll(sc1, b) for b in range(1, B)]).astype(np.float32)
        F = torch_cdfs(np.tile(ends, (B, 1)), mu.ravel(), sc.ravel())
        tab = H.RowTables(*direct_tables(F))
        rows = np.arange(B * L).reshape(B, L)
        states = H.initial_states(B, seed=S)
        sym = rs.randint(0, S, (B, L))
        sym[:, :4] = [0, S - 1, 1, S - 2]
        pad = np.append(ends[0], 1e300)[None] if shared else H.pad_big(ends)
        ers = 0 if shared else S
        want = H.Stacks.from_lists(states, cap=1 << 15)
        ss, got = direct_level(True, pad, mu, sc, S, states, ers=ers)
        want_sym = H.pop(tab, rows, want)
        H.assert_same(f"S={S} {label} pop", got, ss.export(), want_sym, want)
        after = ss.export_lists()
        ss, _ = direct_level(False, pad, mu, sc, S, after, sym=sym, ers=ers)
        H.push(tab, rows, want, sym)
        H.assert_same(f"S={S} {label} push", None, ss.export(), None, want)


# ---- (c) the codec ------------------------------------------------------------------------------------------------------
def _codec(cfg, B, precision, coder="direct", lanes=2, **kw):
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    pc = PipelinedCodec(cfg, sd, Bins(cfg, zend, zcen), B, lanes=lanes, tc_precision=precision, coder=coder, **kw)
    return sd, zend, zcen, pc


RECURSIONS = [("tiny", None), ("tiny3", None), ("cifar8", 10), ("cifar8", 12), ("mnist2", None)]


@pytest.mark.parametrize("precision", ["split", "bf16"])
@pytest.mark.parametrize("name,q", RECURSIONS, ids=[f"{n}-q{q}" if q else n for n, q in RECURSIONS])
def test_recursion_vs_direct_oracle(name, q, precision):
    """Every stream of Bit-Swap and BB-ANS equals the oracle recursion with direct tables driven by the same GPU nets; the
    round trip restores pixels and initial states."""
    cfg = preset(name) if q is None else with_(preset(name), quantbits=q)
    B = 4
    sd, zend, zcen, pc = _codec(cfg, B, precision)
    assert pc.coder == "direct" and all(c.coder == "direct" for c in pc.codecs)
    imgs = synthetic.synthetic_images(cfg, B, seed=31)
    w, head = synthetic.initial_words(20000, seed=100)
    orc = gpu_oracle(cfg, pc.models[0], sd, zend, zcen, cls=DirectOracle)
    for scheme in (BITSWAP, BBANS):
        ss = StreamSet(B, 1 << 15)
        ss.fill(w, head)
        init = ss.export_lists()
        pc.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
        torch.cuda.synchronize()
        ss.raise_on_error()
        got = ss.export_lists()
        enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
        for b in range(B):
            assert got[b] == enc(O.CState(w, head), imgs[b]).to_list(), f"{name} {precision} scheme {scheme}: stream {b}"
        out = pc.decode(ss, B, scheme=scheme)
        torch.cuda.synchronize()
        ss.raise_on_error()
        assert np.array_equal(out.cpu().numpy(), imgs) and ss.export_lists() == init


def _encode_states(codec, cfg, imgs, scheme, w, head):
    ss = StreamSet(imgs.shape[0], 1 << 15)
    ss.fill(w, head)
    codec.encode(ss, torch.from_numpy(imgs).cuda(), scheme=scheme)
    torch.cuda.synchronize()
    ss.raise_on_error()
    return ss.export_lists()


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS], ids=["bitswap", "bbans"])
def test_overlap_mode_and_batch_splits(scheme):
    """Overlap mode equals program order; 3 lanes, 1 lane and a lone BitSwapCodec give the same streams; a batch coded as
    two calls equals one call."""
    cfg = preset("cifar8")
    B = 24
    sd, zend, zcen, pc3 = _codec(cfg, B, "split", lanes=3)
    imgs = synthetic.synthetic_images(cfg, B, seed=8)
    w, head = synthetic.initial_words(20000, seed=100)
    want = _encode_states(pc3, cfg, imgs, scheme, w, head)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=True).load_state_dict(sd)
    m.compress()
    one = BitSwapCodec(cfg, m, pc3.bins, B, coder="direct")
    assert _encode_states(one, cfg, imgs, scheme, w, head) == want, "a lone codec differs from three lanes"
    one.set_dual_stream(True)
    assert _encode_states(one, cfg, imgs, scheme, w, head) == want, "overlap mode differs from program order"
    one.set_dual_stream(False)
    ss = StreamSet(B, 1 << 15)
    ss.fill(w, head)
    x = torch.from_numpy(imgs).cuda()
    one.encode(ss, x[:7].contiguous(), first=0, scheme=scheme)
    one.encode(ss, x[7:].contiguous(), first=7, scheme=scheme)
    torch.cuda.synchronize()
    assert ss.export_lists() == want, "a batch split into two calls differs"
    ref = _encode_states(BitSwapCodec(cfg, m, pc3.bins, B), cfg, imgs, scheme, w, head)
    assert ref != want, "the direct and reference coders gave the same streams"


def test_containers_regions_archives_and_the_other_coder():
    """Edge-coded multi-chain containers, region decodes and an archive round-trip with a direct codec; an archive decoded
    with the other coder fails its initial-state check, both ways."""
    cfg = preset("tiny3")
    rs = np.random.RandomState(9)
    images = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(28, 28), (1, 1), (33, 65), (100, 70), (64, 31)]]
    sd, zend, zcen, dc = _codec(cfg, 16, "split", free_running=True)
    ref = PipelinedCodec(cfg, sd, dc.bins, 16, lanes=2)
    conts = compress_images(dc, images, excess_state_len=3000, edges="code", chain_blocks=2)
    for img, rec in zip(images, decompress_images(dc, conts, channels=3)):
        assert rec.shape == img.shape and np.array_equal(rec, img), img.shape
    regions = [(2, 5, 7, 20, 40), (3, 64, 0, 36, 70), (4, 0, 0, 64, 31), (0, 27, 27, 1, 1)]
    for (i, y, x, h, w), got in zip(regions, decompress_regions(dc, conts, regions, channels=3)):
        assert np.array_equal(got, images[i][y:y + h, x:x + w])
    archives = {}
    for tag, pc in (("direct", dc), ("reference", ref)):
        archives[tag] = compress_archive(pc, images, chain_blocks=3, excess_state_len=3000)
        back = decompress_archive(pc, archives[tag])
        assert all(np.array_equal(b, im) for b, im in zip(back, images)), tag
    assert not np.array_equal(archives["direct"], archives["reference"])
    with pytest.raises(ValueError, match="decoded to a state other than the initial one"):
        decompress_archive(ref, archives["direct"])
    with pytest.raises(ValueError, match="decoded to a state other than the initial one"):
        decompress_archive(dc, archives["reference"])


def test_refusals():
    cfg = preset("tiny")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    m = Model.from_config(cfg, max_batch=2).load_state_dict(sd)
    m.compress()
    bins = Bins(cfg, zend, zcen)
    c = BitSwapCodec(cfg, m, bins, 2, coder="direct")
    with pytest.raises(ValueError, match="set_two_phase"):
        c.set_two_phase(False)
    c.set_two_phase(True)
    with pytest.raises(BswError, match="BSW_E_INVALID"):
        check(lib().bsw_codec_set_two_phase(c._h, 0))
    for bad in (2, -1):
        with pytest.raises(BswError, match="BSW_E_INVALID"):
            check(lib().bsw_codec_set_coder(c._h, bad))
    check(lib().bsw_codec_set_coder(c._h, 0))                       # back to the reference coder: the fused one is allowed
    check(lib().bsw_codec_set_two_phase(c._h, 0))
    check(lib().bsw_codec_set_two_phase(c._h, 1))
    # level entry points: bits other than 31, a support the pop cannot chunk, a short endpoint row stride, small scratch
    S, L, B = 64, 4, 2
    ends, mu, sc = H.level_case(L, S, 6, B, seed=1)
    states = H.initial_states(B, seed=2, n=100)
    e = torch.from_numpy(H.pad_big(ends)).cuda()
    dmu, dsc = torch.from_numpy(mu).cuda(), torch.from_numpy(sc).cuda()
    out = torch.zeros((B, L), dtype=torch.int16, device="cuda")
    nbytes = int(lib().bsw_logistic_scratch_bytes(B, L, S, 0))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ss = StreamSet(B, 1024)
    ss.import_lists(states)
    base = dict(bits=31, S=S, ers=S, nbytes=nbytes)
    for bad in (dict(bits=30), dict(S=48), dict(ers=S - 1), dict(nbytes=nbytes // 4)):
        a = {**base, **bad}
        for fn in (lib().bsw_direct_pop, lib().bsw_direct_push):
            with pytest.raises(BswError, match="BSW_E_INVALID"):
                check(fn(ss.handle, 0, B, dmu.data_ptr(), L, dsc.data_ptr(), L, e.data_ptr(), a["ers"], out.data_ptr(), L,
                         a["S"], a["bits"], 6, scratch.data_ptr(), a["nbytes"], cuda_stream_ptr()))
    assert ss.export_lists() == states
