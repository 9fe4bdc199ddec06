"""Stamps on the GPU: bsw_digest against its numpy twin, the model and bins digests (equal wherever the bitstreams are
equal, different after a one-ulp change), the fingerprint, stamped writers against unstamped ones, and every mismatch
refused by every decoder before a stream is made or a block decoded."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from codec_harness import random_images, setup                                          # noqa: E402
from stamp_harness import digest, hexdigest                                              # noqa: E402
from bitswap_b200 import container, synthetic                                            # noqa: E402
from bitswap_b200._lib import check, lib                                                 # noqa: E402
from bitswap_b200.codec import BBANS, BITSWAP, BitSwapCodec, Bins, PipelinedCodec, device_digest   # noqa: E402
from bitswap_b200.config import preset, with_                                            # noqa: E402
from bitswap_b200.container import (compress_archive, compress_images, decompress_archive, decompress_images,   # noqa: E402
                                    decompress_regions, plan_archive, plan_regions, read_stamp, unpack_container)
from bitswap_b200.model import Model                                                     # noqa: E402

B = 8
N_INIT = 3000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n", [0, 1, 7, 8, 9, 65535, 65536, 65537, 64 << 20])
def test_device_digest_equals_the_twin(n):
    data = np.random.RandomState(n % 1000).randint(0, 256, n).astype(np.uint8)
    t = torch.from_numpy(data).cuda()
    assert device_digest(t) == hexdigest(digest(data.tobytes()))
    if n >= 16:                                                                            # an offset view: same bytes
        assert device_digest(torch.from_numpy(data[8:]).cuda()) == device_digest(t[8:].contiguous())


def _model(cfg, sd, **kw):
    m = Model.from_config(cfg, **kw).load_state_dict(sd)
    m.compress()
    return m


def _fold(v, gain, loggain):
    """The host-side weight-norm fold of bsw_model_load_conv for one output channel, in float32 as it is done there."""
    v = np.asarray(v, dtype=np.float32)
    vnorm = np.float32(np.sqrt(np.sum(v.astype(np.float64) ** 2)))
    g = np.float32(max(float(gain), 0.0) + np.log1p(np.exp(-abs(float(gain))))) if loggain else np.float32(gain)
    return v * (g / (vnorm + np.float32(1e-10)))


def _ulp(sd, key, index=0):
    """A copy of state dict sd with one element of sd[key] moved up by one ulp.  For a conv's v, the first element from
    `index` on whose change survives the fold (a change that rounds away leaves the weights the kernels read as they were)."""
    sd = {k: v.clone() for k, v in sd.items()}
    flat = sd[key].view(-1)
    up = lambda x: torch.nextafter(x, torch.tensor(float("inf"), dtype=x.dtype))          # noqa: E731
    if key.endswith(".v"):
        per = flat.numel() // sd[key].shape[0]
        gain = sd[key[:-2] + ".gain"].view(-1)
        loggain = not key[:-2].endswith(".conv2")
        for i in range(index, flat.numel()):
            o = i // per
            row = flat[o * per:(o + 1) * per].clone()
            row[i - o * per] = up(row[i - o * per])
            if not np.array_equal(_fold(row.numpy(), gain[o].item(), loggain),
                                  _fold(flat[o * per:(o + 1) * per].numpy(), gain[o].item(), loggain)):
                index = i
                break
    flat[index] = up(flat[index])
    return sd


def test_model_digest_is_the_weights_and_only_the_weights():
    cfg = preset("tiny")
    sd = synthetic.synthetic_state_dict(cfg, seed=50, varied=True)
    sd["gen_std"].view(-1)[0] = 20.0         # softplus(20) + 1/1020 in float32: a one-ulp change of it survives the fold
    ref = _model(cfg, sd, max_batch=2, use_tensor_cores=True).digest()
    same = [_model(cfg, sd, max_batch=8, use_tensor_cores=True), _model(cfg, sd, max_batch=3, use_tensor_cores=False),
            _model(cfg, sd, max_batch=4, use_tensor_cores=True, tc_precision="bf16")]
    assert all(m.digest() == ref for m in same)
    m = same[0]
    m.load_state_dict(sd)                                                                  # re-created handle
    assert m.digest() == ref
    bins = Bins(cfg, *synthetic.synthetic_bins(cfg, seed=0))
    pc = PipelinedCodec(cfg, sd, bins, 8, lanes=4, use_tensor_cores=True)
    assert [mm.digest() for mm in pc.models] == [ref] * 4
    assert pc.fingerprint().model_digest == ref
    g = sd["gen_std"].view(-1)[0]
    up = np.nextafter(np.float32(20.0), np.float32(np.inf))
    folded = [np.float32(np.float32(2 / 255) / np.float32(8)) + np.float32(v) for v in (np.float32(20.0), up)]
    assert g.item() == 20.0 and folded[0] != folded[1]
    for key, index in (("infer_in.1.v", 0), ("gen_mu.0.v", sd["gen_mu.0.v"].numel() - 1), ("gen_std", 0)):
        other = _model(cfg, _ulp(sd, key, index), max_batch=2, use_tensor_cores=True).digest()
        assert other != ref, key
    m.load_state_dict(_ulp(sd, "infer_in.1.v"))                                            # a reload starts afresh
    assert m.digest() != ref


def _ulp_array(a, index):
    a = np.array(a, dtype=np.float64, copy=True)
    a[index] = np.nextafter(a[index], np.inf)
    return a


def test_bins_digest_sees_one_ulp_and_quantbits():
    cfg = preset("tiny")
    zend, zcen = synthetic.synthetic_bins(cfg, seed=0)
    zend, zcen = np.asarray(zend), np.asarray(zcen)
    ref = Bins(cfg, zend, zcen).digest()
    assert Bins(cfg, zend, zcen).digest() == ref
    assert Bins(cfg, _ulp_array(zend, (1, 100, 17)), zcen).digest() != ref
    assert Bins(cfg, zend, _ulp_array(zcen, (0, 3, 5))).digest() != ref
    c10, c12 = with_(cfg, quantbits=10), with_(cfg, quantbits=12)
    assert Bins(c10, *synthetic.synthetic_bins(c10, seed=0)).digest() != Bins(c12, *synthetic.synthetic_bins(c12, seed=0)).digest()


def test_fingerprint_follows_the_coder_and_the_tc_heads_switch():
    s = setup("tiny", B, tc=True)
    fp = s.codec.fingerprint()
    assert (fp.coder, fp.tc_precision, fp.use_tensor_cores, fp.tc_heads, fp.quantbits) == ("reference", "split", True, True, 6)
    assert fp.revision == lib().bsw_bitstream_revision() == 1
    assert (fp.model_digest, fp.bins_digest) == (s.model.digest(), s.bins.digest())
    check(lib().bsw_codec_set_coder(s.codec._h, 1))
    assert s.codec.fingerprint() == fp._replace(coder="direct")
    check(lib().bsw_codec_set_coder(s.codec._h, 0))
    assert s.codec.fingerprint() == fp
    s.codec.set_two_phase(False)                                                           # result-neutral: not in it
    s.codec.set_dual_stream(True)
    assert s.codec.fingerprint() == fp
    assert setup("tiny", B, tc=False).codec.fingerprint() == fp._replace(use_tensor_cores=False, tc_heads=False)
    child = ("import sys; sys.path.insert(0, 'tests'); from codec_harness import setup; "
             "print(tuple(setup('tiny', 8, tc=True).codec.fingerprint()))")
    r = subprocess.run([sys.executable, "-c", child], cwd=ROOT, env=dict(os.environ, BSW_TC_HEADS="0"),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip().splitlines()[-1] == repr(tuple(fp._replace(tc_heads=False)))


# ---- stamped writers --------------------------------------------------------------------------------------------------------
def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, tuple):
            _same(x, y)
        else:
            assert np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y


@pytest.mark.parametrize("scheme", [BITSWAP, BBANS])
def test_stamped_output_is_the_unstamped_output_and_the_stamp(scheme):
    s = setup("tiny", B, tc=True)
    fp = s.codec.fingerprint()
    images = random_images(1, [(64, 96), (33, 70), (100, 40)], seed=81)
    for kw in (dict(), dict(chain_blocks=2), dict(edges="code"), dict(edges="code", chain_blocks=3), dict(hwc_quirk=True)):
        hwc = kw.get("hwc_quirk", False)
        plain = compress_images(s.codec, images, excess_state_len=N_INIT, scheme=scheme, **kw)
        stamped = compress_images(s.codec, images, excess_state_len=N_INIT, scheme=scheme, stamp=True, **kw)
        for p, c in zip(plain, stamped):
            assert np.array_equal(c[:p.size], p) and c.size == p.size + 29
            assert read_stamp(c) == container.Stamp(fp, scheme, hwc, N_INIT, 100)
            _same(unpack_container(c, hwc), unpack_container(p, hwc))
        back = decompress_images(s.codec, stamped, channels=1, scheme=scheme, hwc_quirk=hwc)
        want = decompress_images(s.codec, plain, channels=1, scheme=scheme, hwc_quirk=hwc)
        assert all(np.array_equal(b, w) for b, w in zip(back, want))
        regions = [(0, 10, 20, 30, 40), (2, 0, 0, 32, 32)]
        _same(plan_regions(stamped, regions, hwc), plan_regions(plain, regions, hwc))
        for b, w in zip(decompress_regions(s.codec, stamped, regions, channels=1, scheme=scheme, hwc_quirk=hwc),
                        decompress_regions(s.codec, plain, regions, channels=1, scheme=scheme, hwc_quirk=hwc)):
            assert np.array_equal(b, w)
    for L in (None, 3):
        a = compress_archive(s.codec, images, chain_blocks=L, scheme=scheme, excess_state_len=N_INIT)
        a_s = compress_archive(s.codec, images, chain_blocks=L, scheme=scheme, excess_state_len=N_INIT, stamp=True)
        assert np.array_equal(a_s[:a.size], a) and a_s.size == a.size + 29
        assert read_stamp(a_s) == container.Stamp(fp, scheme, False, N_INIT, 100)
        _same(plan_archive(a_s), plan_archive(a))
        back = decompress_archive(s.codec, a_s)
        assert all(np.array_equal(b, im) for b, im in zip(back, images))


# ---- refusals ---------------------------------------------------------------------------------------------------------------
class _Spy:
    """Codec proxy counting decode calls."""

    def __init__(self, codec):
        self.codec, self.calls = codec, 0

    def __getattr__(self, name):
        return getattr(self.codec, name)

    def decode(self, *a, **k):
        self.calls += 1
        return self.codec.decode(*a, **k)


def _tamper(arr, name, value):
    """arr with stamp field `name` set to `value` (the fingerprint's first 14 fields, then scheme / hwc_quirk)."""
    names = list(container.Fingerprint._fields[:14]) + ["d"] * 8 + ["scheme", "hwc_quirk", "excess_state_len", "seed"]
    arr = arr.copy()
    arr[names.index(name) - 29] = value
    return arr


def test_every_mismatch_is_refused_before_any_decoding(monkeypatch):
    s = setup("tiny", B, tc=True)
    cfg, sd = s.cfg, s.sd
    images = random_images(1, [(64, 64), (32, 96)], seed=83)
    cs = compress_images(s.codec, images, excess_state_len=N_INIT, stamp=True)
    a_s = compress_archive(s.codec, images, chain_blocks=2, excess_state_len=N_INIT, stamp=True)
    made = []
    real = container.StreamSet
    monkeypatch.setattr(container, "StreamSet", lambda *a, **k: made.append(1) or real(*a, **k))

    def codec_of(model=None, bins=None, c=cfg, **kw):
        return BitSwapCodec(c, model or s.model, bins or s.bins, B, **kw)
    zend = _ulp_array(s.zend, (0, 2, 9))
    c7 = with_(cfg, quantbits=7)
    tiny3 = preset("tiny3")
    cases = [
        ("coder", codec_of(coder="direct"), {}),
        ("tc_precision", codec_of(_model(cfg, sd, max_batch=B, use_tensor_cores=True, tc_precision="bf16")), {}),
        ("use_tensor_cores", codec_of(_model(cfg, sd, max_batch=B, use_tensor_cores=False)), {}),
        ("reswidth", BitSwapCodec(tiny3, _model(tiny3, synthetic.synthetic_state_dict(tiny3, seed=50), max_batch=B),
                                  Bins(tiny3, *synthetic.synthetic_bins(tiny3, seed=0)), B), {}),
        ("quantbits", codec_of(bins=Bins(c7, *synthetic.synthetic_bins(c7, seed=0)), c=c7), {}),
        ("model_digest", codec_of(_model(cfg, _ulp(sd, "gen_mu.0.v"), max_batch=B, use_tensor_cores=True)), {}),
        ("bins_digest", codec_of(bins=Bins(cfg, zend, s.zcen)), {}),
        ("scheme", s.codec, dict(scheme=BBANS)),
        ("hwc_quirk", s.codec, dict(hwc_quirk=True)),
        ("revision", s.codec, dict(revision=7)),
    ]
    for field, codec, how in cases:
        spy = _Spy(codec)
        if "revision" in how:
            cont, arch, args = [_tamper(c, "revision", 7) for c in cs], _tamper(a_s, "revision", 7), {}
        elif field in ("scheme", "hwc_quirk"):                  # an archive takes neither as an argument: its stamp is tampered
            cont, arch, args = cs, _tamper(a_s, field, 1), how
        else:
            cont, arch, args = cs, a_s, {}
        calls = [lambda: decompress_images(spy, cont, channels=1, **args),
                 lambda: decompress_regions(spy, cont, [(1, 0, 40, 8, 8)], channels=1, **args),
                 lambda: decompress_archive(spy, arch)]
        for i, call in enumerate(calls):
            try:
                call()
            except ValueError as e:
                assert f"{field}: stamped" in str(e) or field in str(e) and i == 2, (field, i, str(e))
            else:
                raise AssertionError(f"{field}: decoder {i} did not refuse")
        assert spy.calls == 0 and not made, field
    back = decompress_images(_Spy(s.codec), cs, channels=1)                               # the matching codec decodes
    assert all(np.array_equal(b, im) for b, im in zip(back, images)) and made


def test_a_stamped_container_gets_the_initial_state_check():
    s = setup("tiny", B, tc=True)
    (img,) = random_images(1, [(64, 64)], seed=85)
    (c,) = compress_images(s.codec, [img], excess_state_len=N_INIT)
    (cs,) = compress_images(s.codec, [img], excess_state_len=N_INIT, stamp=True)
    assert np.array_equal(decompress_images(s.codec, [cs], channels=1)[0], img)
    bad, bad_s = c.copy(), cs.copy()
    bad[-5] ^= 1                                                                           # head_lo of the one chain
    bad_s[c.size - 5] ^= 1
    with pytest.raises(ValueError, match="decoded to a state other than the initial one"):
        decompress_images(s.codec, [bad_s], channels=1)
    (got,) = decompress_images(s.codec, [bad], channels=1)                                 # unstamped: no check, as before
    assert got.shape == img.shape
