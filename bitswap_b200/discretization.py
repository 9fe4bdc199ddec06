"""Latent-space discretisation with the reference's signature, computed on the GPU.

Reference: discretize() / discretize_kbins(), discretization.py:9-118.  For every latent level it draws
30 * 2^q samples per dimension from the generative chain (ancestral sampling down from the Logistic(0,1)
prior) and from the inference chain (up from training images), keeps them in float16, and fits 2^q
uniform-width bins per dimension between the sample extrema (sklearn KBinsDiscretizer(strategy='uniform'),
whose bin_edges_ are exactly np.linspace(min, max, n_bins + 1) per feature).  The top level uses the
equal-mass bins of the prior (rand.Bins on float32 zeros/ones).

Differences from the reference, by necessity of the offline setting: the training images are an argument
(`images`, uint8 [N, C, 32, 32]) instead of a torchvision download, and the uniform-width fit is a running min/max
kept by the sampling kernel (csrc/discretize.cu) + np.linspace arithmetic on the device instead of sklearn
(tests/test_discretization_cpu.py pins `uniform_bins`, the host statement of the same fit, against sklearn; the GPU
test pins the kernels against `uniform_bins` and the whole procedure against a torch-CPU run of the same nets fed the same noise).
The returned tensors have the reference's layout and dtype handling: (zendpoints [nz, zdim, 2^q - 1],
zcentres [nz, zdim, 2^q]) cast to `type` on `device` (discretization.py:99).
"""
import numpy as np
import torch

from .rand import Bins


def logistic_eps(shape, device, bound=1e-5, generator=None):
    """Logistic(0,1) noise by inverse-cdf of clamped uniforms (utils/torch/rand.py:11-20)."""
    u = torch.rand(shape, device=device, generator=generator)
    u = torch.clamp(u, min=bound, max=1 - bound)
    return torch.log(u) - torch.log1p(-u)


def uniform_bins(samples, quantbits):
    """samples [n, dim] -> (endpoints [dim, 2^q - 1], centres [dim, 2^q]) float64: equal-width bins between the
    per-dimension extrema (discretize_kbins with strategy='uniform', discretization.py:105-118)."""
    s = torch.as_tensor(samples).double()
    lo, hi = s.min(dim=0).values, s.max(dim=0).values
    n = 1 << quantbits
    steps = torch.arange(n + 1, dtype=torch.float64, device=s.device)
    # np.linspace semantics (sklearn builds the edges with it): start + k*step, last point forced to stop
    edges = lo[:, None] + steps[None, :] * ((hi - lo) / n)[:, None]
    edges[:, -1] = hi
    centres = (edges[:, :-1] + edges[:, 1:]) / 2
    return edges[:, 1:-1].contiguous(), centres.contiguous()


@torch.no_grad()
def discretize(nz, quantbits, type, device, model, dataset, images=None, ppb=30, bs=128, seed=0, uniforms=None):
    """Same positional signature as the reference.  `model` is a bitswap_b200.model.Model with max_batch >= bs;
    `images`: uint8 tensor [N, C, 32, 32] standing in for the dataset named by `dataset`.
    `uniforms(tag, shape)` (optional) supplies the U(0,1) draws as float32 CUDA tensors (tests feed a CPU run the same
    noise); default: torch's CUDA generator seeded with `seed`.

    Per batch ONE kernel (bsw_discretize_sample) turns (mu, scale, u) into the float16 samples the next net reads and folds
    them into per-dimension running extrema; the equal-width fit (bsw_discretize_edges) then needs no pass over the
    2 * ppb * 2^q * zdim samples of a level."""
    from ._lib import lib, check, cuda_stream_ptr
    from .codec import check_quantbits
    check_quantbits(quantbits)                          # 1..12, before any device work
    assert images is not None, "offline: pass the training images explicitly (the reference downloads them)"
    cfg = model.cfg
    assert cfg.nz == nz
    zdim = cfg.zdim
    nbins = 1 << quantbits
    nsamples = ppb * nbins
    batches = nsamples // bs
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if uniforms is None:
        def uniforms(tag, shape):
            return torch.rand(shape, device="cuda", generator=gen)
    zendpoints = torch.zeros((nz, zdim, nbins - 1), dtype=torch.float64)
    zcentres = torch.zeros((nz, zdim, nbins), dtype=torch.float64)
    top = Bins(torch.zeros((1, 1, zdim)), torch.ones((1, 1, zdim)), quantbits)          # float32, as :25-27
    zendpoints[nz - 1] = top.endpoints()[0, 0].double()
    zcentres[nz - 1] = top.centres()[0, 0].double()
    if nz == 1:
        return zendpoints.type(type).to(device), zcentres.type(type).to(device)
    model.compress(True)
    imgs = images.to("cuda").float().reshape(images.shape[0], -1)
    imgs = (imgs - 127.5) / 127.5            # compressing-mode nets take centred inputs (cifar_train.py:330-333)
    while imgs.shape[0] < nsamples:
        imgs = torch.cat([imgs, imgs])
    gen_s = torch.zeros((nz, nsamples, zdim), dtype=torch.float16, device="cuda")         # float16 storage, :59-61
    inf_s = torch.zeros((nz, nsamples, zdim), dtype=torch.float16, device="cuda")
    u_top = torch.clamp(uniforms(("top",), (nsamples, zdim)), min=1e-30, max=1 - 1e-30)
    gen_s[-1] = (torch.log(u_top) - torch.log1p(-u_top)).half()                           # :60 logistic_eps(bound=1e-30)
    mm = torch.empty((nz - 1, 2 * zdim), dtype=torch.int32, device="cuda")                # running extrema per level
    for lv in range(nz - 1):
        check(lib().bsw_discretize_reset(mm[lv].data_ptr(), zdim, cuda_stream_ptr()))
    used = batches * bs
    if used < nsamples:          # the reference fits over its whole zero-initialised sample arrays (:59-61,82)
        zero_row = torch.zeros((1, zdim), dtype=torch.float16, device="cuda")
        for lv in range(nz - 1):
            check(lib().bsw_discretize_fold(zero_row.data_ptr(), mm[lv].data_ptr(), 1, zdim, cuda_stream_ptr()))

    def draw(tag, mu, scale, out, level):
        u = uniforms(tag, tuple(mu.shape)).float().contiguous()
        mu, scale = mu.float().contiguous(), scale.float().contiguous()
        check(lib().bsw_discretize_sample(mu.data_ptr(), scale.data_ptr(), zdim, u.data_ptr(), 1e-30, out.data_ptr(),
                                          mm[level].data_ptr(), mu.shape[0], zdim, cuda_stream_ptr()))

    for zi in reversed(range(1, nz)):                                                     # :64-78
        for bi in range(batches):
            sl = slice(bi * bs, bi * bs + bs)
            mu, scale = model.generate(zi)(given=gen_s[zi][sl].float())
            draw(("gen", zi, bi), mu, scale, gen_s[zi - 1][sl], zi - 1)
        lvl = nz - zi - 1
        for bi in range(batches):
            sl = slice(bi * bs, bi * bs + bs)
            given = imgs[sl] if lvl == 0 else inf_s[lvl - 1][sl].float()
            mu, scale = model.infer(lvl)(given=given)
            draw(("inf", lvl, bi), mu, scale, inf_s[lvl][sl], lvl)
    ze = torch.empty((nz - 1, zdim, nbins - 1), dtype=torch.float64, device="cuda")
    zc = torch.empty((nz - 1, zdim, nbins), dtype=torch.float64, device="cuda")
    for zi in range(nz - 1):                                                              # :81-83
        check(lib().bsw_discretize_edges(mm[zi].data_ptr(), zdim, quantbits, ze[zi].data_ptr(), nbins - 1, zc[zi].data_ptr(), nbins,
                                         cuda_stream_ptr()))
    torch.cuda.synchronize()
    zendpoints[:nz - 1], zcentres[:nz - 1] = ze.cpu(), zc.cpu()
    return zendpoints.type(type).to(device), zcentres.type(type).to(device)
