"""GPU parity for the VQ-VAE: encode -> bit-exact int64 codes, decode -> waveform, against the reference's
outputs (tests/golden) and the oracle; argmin kernel unit tests incl. ties and ragged sizes."""
import numpy as np
import pytest
import torch

from golden_util import Fixture, rel_err
from oracle.vqvae_np import quantise

pytestmark = pytest.mark.gpu


def _make(fx):
    from jukebox_b200.hparams import setup_hparams
    from jukebox_b200.make_models import make_vqvae
    c = fx.cfg
    vq = make_vqvae(setup_hparams(c["hps_name"], dict(restore_vqvae="", **c["overrides"])), "cpu")
    vq.load_state_dict({k: torch.from_numpy(v) for k, v in fx.weights().items()}, strict=True)
    return vq.cuda().eval()


@pytest.mark.parametrize("tag", ["small", "3level"])
def test_encode_decode_match_reference(tag):
    fx = Fixture(f"vqvae_{tag}")
    c = fx.cfg
    vq = _make(fx)
    x = torch.from_numpy(fx["x"]).cuda()
    bs = x.shape[0]
    with torch.no_grad():
        zs = vq.encode(x, bs_chunks=bs)
        lat = [vq.encoders[l](vq.preprocess(x))[-1] for l in range(c["levels"])]
    for l in range(c["levels"]):
        ref_lat = np.transpose(fx[f"lat{l}"], (0, 2, 1))           # reference is NCT
        assert rel_err(lat[l].cpu().numpy(), ref_lat) < 2e-5
        assert zs[l].dtype == torch.int64 and tuple(zs[l].shape) == fx[f"z{l}"].shape
        z, zref = zs[l].cpu().numpy(), fx[f"z{l}"]
        mism = np.argwhere(z != zref)
        if len(mism):        # a flip is only acceptable on a numerical near-tie of the reference's distances
            flat = ref_lat.reshape(-1, ref_lat.shape[-1])
            _, dist = quantise(flat, fx.weights()[f"bottleneck.level_blocks.{l}.k"])
            d = dist.reshape(*zref.shape, -1)
            for n, t in mism:
                gap = abs(d[n, t, z[n, t]] - d[n, t, zref[n, t]])
                assert gap < 1e-4 * abs(d[n, t, zref[n, t]]), (l, n, t, gap)
        print(f"vqvae_{tag} level {l}: {len(mism)} / {z.size} code mismatches")
        assert len(mism) <= max(1, z.size // 2000)
        with torch.no_grad():
            xd = vq.decode([torch.from_numpy(zref).cuda() for _ in range(1)] +
                           [torch.from_numpy(fx[f"z{k}"]).cuda() for k in range(l + 1, c["levels"])],
                           start_level=l, bs_chunks=bs)
        assert tuple(xd.shape) == fx[f"xd{l}"].shape
        e = rel_err(xd.cpu().numpy(), fx[f"xd{l}"])
        print(f"vqvae_{tag} level {l}: decode rel err {e:.2e}")
        assert e < 2e-5


@pytest.mark.parametrize("n,kbins,width", [(1, 7, 64), (63, 128, 64), (64, 129, 64), (1000, 2048, 64), (257, 50, 32)])
def test_argmin_matches_oracle(n, kbins, width):
    from jukebox_b200.vqvae.bottleneck import BottleneckBlock
    rng = np.random.RandomState(n)
    x = rng.standard_normal((n, width)).astype(np.float32)
    k = rng.standard_normal((kbins, width)).astype(np.float32)
    blk = BottleneckBlock(kbins, width, 0.99).cuda()
    blk.k.copy_(torch.from_numpy(k))
    idx, dist = blk.quantise(torch.from_numpy(x).cuda())
    ref, d = quantise(x, k)
    idx = idx.cpu().numpy()
    bad = np.nonzero(idx != ref)[0]
    for i in bad:
        assert abs(d[i, idx[i]] - d[i, ref[i]]) < 1e-5 * abs(d[i, ref[i]])
    assert len(bad) <= max(1, n // 1000)
    assert np.allclose(dist.cpu().numpy(), d.min(-1), rtol=1e-4, atol=1e-4)


def test_argmin_ties_pick_lowest_index_and_gather_roundtrip():
    from jukebox_b200.vqvae.bottleneck import BottleneckBlock
    kbins, width = 300, 64
    rng = np.random.RandomState(0)
    k = rng.standard_normal((kbins, width)).astype(np.float32)
    k[150] = k[3]
    k[299] = k[3]                       # exact duplicates: torch/numpy argmin return the first
    blk = BottleneckBlock(kbins, width, 0.99).cuda()
    blk.k.copy_(torch.from_numpy(k))
    x = torch.from_numpy(k[[3, 150, 299, 7]]).cuda()
    idx, _ = blk.quantise(x)
    assert idx.tolist() == [3, 3, 3, 7]
    # dequantise(quantise(codebook rows)) is the identity on distinct rows (idempotence)
    codes = torch.arange(kbins, device="cuda").view(1, -1)
    back = blk.encode(blk.decode(codes))
    expect = codes.clone()
    expect[0, 150] = 3
    expect[0, 299] = 3
    assert torch.equal(back, expect)
    assert blk.encode(torch.zeros(2, 0, width, device="cuda")).shape == (2, 0)


def test_decode_is_batch_independent_and_linear_in_out_bias():
    """size-independent properties at a larger size: chunked == unchunked decode; per-sample independence"""
    fx = Fixture("vqvae_3level")
    vq = _make(fx)
    g = torch.Generator(device="cuda").manual_seed(0)
    zs = [torch.randint(0, vq.l_bins, (4, 4096 // int(h)), device="cuda", generator=g) for h in vq.hop_lengths / vq.hop_lengths[0]]
    with torch.no_grad():
        a = vq.decode(zs[1:], start_level=1, bs_chunks=1)
        b = vq.decode(zs[1:], start_level=1, bs_chunks=4)
        c = vq.decode([z[2:3] for z in zs[1:]], start_level=1)
    assert torch.equal(a, b)
    assert torch.equal(a[2:3], c)


@pytest.mark.parametrize("C,dil,T", [(64, 1, 1000), (64, 2187, 5000), (32, 27, 777), (32, 1, 64), (64, 9, 65),
                                     (64, 27, 128), (32, 243, 4101), (64, 729, 20000), (32, 3, 129)])
def test_tensor_core_resblock_matches_exact_fma_kernel(C, dil, T):
    """jk_resblock_tc (split-precision tensor-core block, decoder side) against jk_resblock_cl (exact fp32 FMAs): same block
    (resnet.py:27-44), fp32-level agreement; ragged T, dilations beyond the tile, both channel counts.  T >= 128 runs the
    wgmma / TMA kernel (vqvae_t5.cu: 128-position MMA tiles, out-of-range rows zero-filled by the tensor map), shorter
    clips (T = 64, 65) the fp16 x 3 mma.sync kernel"""
    import ctypes as Cc
    from jukebox_b200._lib import lib, check, ptr, stream_ptr
    g = torch.Generator(device="cuda").manual_seed(C + dil)
    n = 2
    x = torch.randn(n, T, C, device="cuda", generator=g)
    w1 = torch.randn(3, C, C, device="cuda", generator=g) / (3 * C) ** 0.5
    w2 = torch.randn(1, C, C, device="cuda", generator=g) / C ** 0.5
    b1 = torch.randn(C, device="cuda", generator=g) * 0.1
    b2 = torch.randn(C, device="cuda", generator=g) * 0.1
    exact, tc = torch.empty_like(x), torch.empty_like(x)
    check(lib().jk_resblock_cl(ptr(x), ptr(exact), None, ptr(w1), ptr(b1), ptr(w2), ptr(b2), n, T, C, C, dil, 0.7, stream_ptr()))
    check(lib().jk_resblock_tc(ptr(x), ptr(tc), ptr(w1), ptr(b1), ptr(w2), ptr(b2), n, T, C, dil, 0.7, stream_ptr()))
    ref = x.double() + 0.7 * (torch.einsum("ntc,cd->ntd", torch.relu(
        sum(torch.einsum("ntc,cd->ntd", torch.relu(torch.nn.functional.pad(x.double(), (0, 0, dil, dil))[:, k * dil:k * dil + T]), w1[k].double())
            for k in range(3)) + b1.double()), w2[0].double()) + b2.double())
    e_exact = float((exact.double() - ref).abs().max() / ref.abs().max())
    e_tc = float((tc.double() - ref).abs().max() / ref.abs().max())
    print(f"C {C} dil {dil} T {T}: exact-FMA kernel vs fp64 {e_exact:.1e}, tensor-core kernel vs fp64 {e_tc:.1e}")
    assert e_exact < 2e-6 and e_tc < 4e-6


@pytest.mark.parametrize("kind,ci,co,T", [("k3", 64, 64, 1000), ("k3", 64, 32, 333), ("k3d", 32, 32, 5000), ("up", 64, 64, 777),
                                          ("up", 32, 64, 64), ("down", 32, 64, 1024)])
def test_tensor_core_conv_matches_exact_kernel(kind, ci, co, T):
    """decoder-side convs with tensor_cores set (fp16 x 3 split on mma.sync) against the exact-FMA kernels and torch:
    k3 'same' (dilated too), the two phases of the k4-s2 transposed conv, the strided k4 conv; ragged T"""
    from jukebox_b200.vqvae.ops_cl import Conv1d, ConvTranspose1d
    torch.manual_seed(ci + co + T)
    if kind == "up":
        m = ConvTranspose1d(ci, co, 4, 2, 1)
    elif kind == "down":
        m = Conv1d(ci, co, 4, 2, 1)
    else:
        d = 27 if kind == "k3d" else 1
        m = Conv1d(ci, co, 3, 1, d, d)
    m = m.cuda()
    x = torch.randn(3, T, ci, device="cuda")
    with torch.no_grad():
        exact = m(x)
        m.tensor_cores = True
        tc = m(x)
    # fp64 reference through torch on the same weights
    with torch.no_grad():
        md = {k: v.double() for k, v in m.state_dict().items()}
        xd = x.double().transpose(1, 2)
        if kind == "up":
            ref = torch.nn.functional.conv_transpose1d(xd, md["weight"], md["bias"], stride=2, padding=1)
        elif kind == "down":
            ref = torch.nn.functional.conv1d(xd, md["weight"], md["bias"], stride=2, padding=1)
        else:
            ref = torch.nn.functional.conv1d(xd, md["weight"], md["bias"], padding=d, dilation=d)
        ref = ref.transpose(1, 2)
    assert tc.shape == exact.shape == ref.shape
    e_exact = float((exact.double() - ref).abs().max() / ref.abs().max())
    e_tc = float((tc.double() - ref).abs().max() / ref.abs().max())
    print(f"{kind} {ci}->{co} T {T}: exact kernel vs fp64 {e_exact:.1e}, tensor-core kernel vs fp64 {e_tc:.1e}")
    assert e_exact < 2e-6 and e_tc < 4e-6
