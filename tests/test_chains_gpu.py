"""Images coded as several chains on the GPU: exact round trips, every chain against the oracle's demo procedure on its
blocks, the calls split into sub-ranges of max_batch streams, and mixed single- and multi-chain containers."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from edge_oracle import EdgeOracle                                         # noqa: E402
from oracle import oracle as O                                             # noqa: E402
from bitswap_b200 import synthetic                                         # noqa: E402
from bitswap_b200.config import preset                                     # noqa: E402
from bitswap_b200.model import Model                                       # noqa: E402
from bitswap_b200.codec import BitSwapCodec, Bins, PipelinedCodec, BITSWAP, BBANS   # noqa: E402
from bitswap_b200.streams import StreamSet                                 # noqa: E402
from bitswap_b200.container import (chain_sizes, compress_images, decompress_images, extract_blocks,   # noqa: E402
                                    extract_edge_blocks, unpack_container)

N_INIT = 3000


def _setup(name, B, tc=False, varied=True):
    cfg = preset(name)
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=varied)
    m = Model.from_config(cfg, max_batch=B, use_tensor_cores=tc).load_state_dict(sd)
    m.compress()
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    bins = Bins(cfg, zend, zcen)
    return cfg, m, sd, zend, zcen, bins


def _images(C, sizes, seed):
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, (h, w, C)).astype(np.uint8) for h, w in sizes]


def _tiles(img, edges):
    """(blocks [n, 32, 32, C], extents [n, 2] or None) of an image as compress_images tiles it."""
    if edges == "code":
        blocks, ext, _, _ = extract_edge_blocks(img)
        return blocks, ext
    return extract_blocks(img)[0], None


def _chains_of(cont):
    """[(words, head, nblocks)] of a container, in block order."""
    words, offs, heads, nblocks, _, _ = unpack_container(cont)
    return [(words[offs[k]:offs[k + 1]], int(heads[k]), int(nblocks[k])) for k in range(len(heads))]


def _gpu_oracle(cfg, m, sd, zend, zcen):
    orc = EdgeOracle(cfg, O.ModelOracle(cfg, sd), zend, zcen, coder="c", pmf="cuda")

    def gpu_net(kind, level, given):
        f = m.infer(level) if kind == "infer" else m.generate(level)
        mu, sc = f(given.cuda())
        return mu.cpu(), sc.cpu()
    orc._net = gpu_net
    return orc


def _oracle_chain(orc, blocks, extents, scheme, n_init=N_INIT):
    """The reference demo procedure (demo_compress.py:113-162) run by the oracle on one chain's blocks, from the seeded
    initial state: (the words above the lowest depth any pop reached, head)."""
    wds, head = synthetic.initial_words(n_init, seed=100)
    st = O.CState(wds, head)
    low = st.n
    pops = []
    orc.trace = pops
    enc = orc.encode_image if scheme == BITSWAP else orc.encode_image_bbans
    for k, b in enumerate(blocks):
        st = enc(st, b.transpose(2, 0, 1), extent=None if extents is None else (int(extents[k][0]), int(extents[k][1])))
    orc.trace = None
    low = min([ln - 1 for tag, ln, _ in pops if tag.startswith("pop")] + [low])
    return np.asarray(st.words[low:st.n], dtype=np.uint32), int(st.head)


def _lone_chain(codec, blocks, extents, scheme, n_init=4000):
    """One chain coded on a stream set of its own, one block per call: (the words above the lowest depth, head).  The
    blocks and extents stay on the device until the lanes are joined: a free-running codec reads them on its own streams."""
    wds, head = synthetic.initial_words(n_init, seed=100)
    ss = StreamSet(1, n_init + 1400 * len(blocks) + 64, device=codec.device)
    ss.fill(wds, head)
    x = torch.from_numpy(np.ascontiguousarray(blocks.transpose(0, 3, 1, 2))).cuda()
    e = None if extents is None else torch.from_numpy(np.ascontiguousarray(extents, dtype=np.int16)).cuda()
    for k in range(len(blocks)):
        codec.encode(ss, x[k:k + 1], scheme=scheme, extent=None if e is None else e[k:k + 1])
    if hasattr(codec, "join"):
        codec.join()
    torch.cuda.synchronize()
    ss.raise_on_error()
    words, offs, heads, _ = ss.export()
    return words[ss.min_words()[0]:offs[1]], int(heads[0])


CASES = [("tiny", BITSWAP, "crop"), ("tiny", BBANS, "code"), ("tiny3", BITSWAP, "code"), ("tiny3", BBANS, "crop")]


@pytest.mark.parametrize("name,scheme,edges", CASES)
def test_round_trips_and_every_chain_equals_the_oracle(name, scheme, edges):
    """Odd-sized images at chain_blocks 1, 2, 3 and 7 round-trip exactly; every chain of every container holds what the
    oracle's demo procedure writes for that chain's blocks, driven by the same GPU nets."""
    sizes = [(100, 70), (33, 65), (64, 96), (97, 40)] if edges == "code" else [(100, 70), (64, 96), (130, 33), (32, 32)]
    cfg, m, sd, zend, zcen, bins = _setup(name, 16)
    codec = BitSwapCodec(cfg, m, bins, 16)
    C = cfg.xs[0]
    images = _images(C, sizes, seed=31)
    want = images if edges == "code" else [im[:im.shape[0] // 32 * 32, :im.shape[1] // 32 * 32] for im in images]
    orc = _gpu_oracle(cfg, m, sd, zend, zcen)
    checked = 0
    for L in (1, 2, 3, 7):
        conts = compress_images(codec, images, excess_state_len=N_INIT, scheme=scheme, edges=edges, chain_blocks=L)
        back = decompress_images(codec, conts, channels=C, scheme=scheme)
        for img, rec in zip(want, back):
            assert rec.shape == img.shape and np.array_equal(rec, img), (L, img.shape)
        for img, cont in zip(images, conts):
            blocks, ext = _tiles(img, edges)
            chains = _chains_of(cont)
            assert [nb for _, _, nb in chains] == chain_sizes(len(blocks), L)
            if L not in (1, 3) and img is not images[0]:        # the oracle is slow: every chain of two splits, one image of the others
                continue
            s = 0
            for ws, hd, nb in chains:
                ow, oh = _oracle_chain(orc, blocks[s:s + nb], None if ext is None else ext[s:s + nb], scheme)
                assert np.array_equal(ws, ow) and hd == oh, (L, img.shape, s)
                s += nb
                checked += 1
    assert checked > 0


def test_no_split_writes_the_reference_container():
    """chain_blocks=None and any chain_blocks >= an image's block count write the same arrays as a call without it."""
    cfg, m, sd, zend, zcen, bins = _setup("tiny3", 4)
    codec = BitSwapCodec(cfg, m, bins, 4)
    images = _images(3, [(100, 70), (64, 96), (33, 1)], seed=37)          # 4 x 3, 2 x 3 and 2 x 1 blocks
    for edges in ("crop", "code"):
        imgs = images[:2] if edges == "crop" else images
        plain = compress_images(codec, imgs, excess_state_len=N_INIT, edges=edges)
        for L in (None, 12, 13, 1000):
            got = compress_images(codec, imgs, excess_state_len=N_INIT, edges=edges, chain_blocks=L)
            assert all(a.dtype == b.dtype and np.array_equal(a, b) for a, b in zip(plain, got)), (edges, L)
    # an image of at most L blocks keeps the reference layout next to an image that is split
    mixed = compress_images(codec, images, excess_state_len=N_INIT, edges="code", chain_blocks=6)
    assert len(_chains_of(mixed[0])) == 2 and np.array_equal(mixed[1], plain[1]) and np.array_equal(mixed[2], plain[2])


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_more_chains_than_max_batch(scheme):
    """24 chains through a codec of max_batch 8 (three calls per step) write the containers a codec of max_batch 24 writes
    (one call per step); so does a free-running 4-lane PipelinedCodec of max_batch 8, whose lanes must see every stream
    at the same lane at every step."""
    cfg, m, sd, zend, zcen, bins = _setup("tiny3", 24)
    images = _images(3, [(150, 390), (33, 65)], seed=41)                 # 5 x 13 and 2 x 3 blocks, edge-coded
    big = BitSwapCodec(cfg, m, bins, 24)
    small = BitSwapCodec(cfg, m, bins, 8)
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=4, use_tensor_cores=False, free_running=True)
    kw = dict(excess_state_len=N_INIT, scheme=scheme, edges="code", chain_blocks=3)
    want = compress_images(big, images, **kw)
    assert [[nb for _, _, nb in _chains_of(c)] for c in want] == [[3] * 21 + [2], [3, 3]]   # 24 streams, 23 at the last step
    for codec in (small, pc):
        got = compress_images(codec, images, **kw)
        assert all(np.array_equal(a, b) for a, b in zip(want, got))
        back = decompress_images(codec, got, scheme=scheme)
        assert all(np.array_equal(a, b) for a, b in zip(images, back))


def test_one_call_decodes_single_and_multi_chain_containers():
    cfg, m, sd, zend, zcen, bins = _setup("tiny3", 12)
    codec = BitSwapCodec(cfg, m, bins, 12)
    images = _images(3, [(100, 70), (20, 20), (64, 96), (130, 33)], seed=43)
    single = compress_images(codec, images, excess_state_len=N_INIT, edges="code")
    multi = compress_images(codec, images, excess_state_len=N_INIT, edges="code", chain_blocks=3)
    assert [len(_chains_of(c)) for c in multi] == [4, 1, 2, 4]
    mix = [multi[0], single[1], single[2], multi[2], multi[3], single[0]]
    back = decompress_images(codec, mix)
    for rec, img in zip(back, [images[0], images[1], images[2], images[2], images[3], images[0]]):
        assert np.array_equal(rec, img)


def test_imagenetcrop4_tensor_cores_each_chain_equals_a_lone_chain():
    """The config-5 model on tensor cores through a free-running 2-lane PipelinedCodec: chain k of an edge-coded image
    holds exactly what a lone single-chain encode of its blocks leaves, and the containers round-trip."""
    cfg = preset("imagenetcrop4")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=False)
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=2, use_tensor_cores=True, free_running=True)
    images = _images(3, [(100, 130), (64, 31)], seed=47)                  # 4 x 5 and 2 x 1 blocks
    conts = compress_images(pc, images, excess_state_len=4000, edges="code", chain_blocks=6)
    back = decompress_images(pc, conts)
    assert all(np.array_equal(a, b) for a, b in zip(images, back))
    blocks, ext = _tiles(images[0], "code")
    chains = _chains_of(conts[0])
    assert [nb for _, _, nb in chains] == [5, 5, 5, 5]
    s = 0
    for ws, hd, nb in chains:
        lw, lh = _lone_chain(pc, blocks[s:s + nb], ext[s:s + nb], BITSWAP)
        assert np.array_equal(ws, lw) and hd == lh, s
        s += nb
    assert np.array_equal(conts[1], compress_images(pc, images[1:], excess_state_len=4000, edges="code")[0])
