"""The wide decoder-side convolutions (jk_conv1d_tc_wide: wgmma + TMA, fp16 x 3 split) against float64 torch on the same
weights, next to the exact-FMA kernel they replace: every conv kind of the upsampler Conditioner (k3 'same' with small
and huge dilations, the two phases of the k4-s2 transposed conv), the wide ResConv1DBlock, and whole Conditioners at the
released upsamplers' geometry."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PAIRS = [(1920, 1024), (1024, 1024), (1024, 1920), (512, 512), (1024, 512), (192, 320)]
KINDS = [("k3", 1), ("k3", 27), ("k3", 2187), ("up", 1)]
SIZES = [(128, 3), (1000, 1), (2048, 3), (4101, 1)]


def _err(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


def _module(kind, dil, ci, co):
    from jukebox_b200.vqvae.ops_cl import Conv1d, ConvTranspose1d
    m = ConvTranspose1d(ci, co, 4, 2, 1) if kind == "up" else Conv1d(ci, co, 3, 1, dil, dil)
    return m.cuda()


def _ref64(m, kind, dil, x):
    w, b = m.weight.detach().double(), m.bias.detach().double()
    xd = x.double().transpose(1, 2)
    if kind == "up":
        y = F.conv_transpose1d(xd, w, b, stride=2, padding=1)
    else:
        y = F.conv1d(xd, w, b, padding=dil, dilation=dil)
    return y.transpose(1, 2)


@pytest.mark.parametrize("T,n", SIZES)
@pytest.mark.parametrize("ci,co", PAIRS)
@pytest.mark.parametrize("kind,dil", KINDS)
def test_wide_conv_matches_float64(kind, dil, ci, co, T, n):
    torch.manual_seed(ci + 3 * co + T + dil)
    m = _module(kind, dil, ci, co)
    x = torch.randn(n, T, ci, device="cuda")
    with torch.no_grad():
        exact = m(x)
        m.tensor_cores = True
        tc = m(x)
        ref = _ref64(m, kind, dil, x)
    assert tc.shape == exact.shape == ref.shape
    assert m._split is not None, "the tensor-core route did not take the wide kernel"
    e_exact, e_tc = _err(exact, ref), _err(tc, ref)
    print(f"{kind} d{dil} {ci}->{co} T {T} n {n}: exact kernel vs fp64 {e_exact:.1e}, wide tensor-core kernel vs fp64 {e_tc:.1e}")
    assert e_tc <= max(4e-6, 2 * e_exact)


@pytest.mark.parametrize("res_scale", [1.0, 0.25])
def test_wide_resblock_matches_float64(res_scale):
    from jukebox_b200.vqvae.resnet import ResConv1DBlock, use_tensor_cores
    torch.manual_seed(7)
    blk = ResConv1DBlock(1024, 1024, dilation=27, res_scale=res_scale).cuda()
    x = torch.randn(2, 1000, 1024, device="cuda")
    c3, c1 = blk.model[1], blk.model[3]
    with torch.no_grad():
        exact = blk(x)
        use_tensor_cores(blk)
        tc = blk(x)
        xd = x.double().transpose(1, 2)
        h = F.conv1d(F.relu(xd), c3.weight.double(), c3.bias.double(), padding=27, dilation=27)
        h = F.conv1d(F.relu(h), c1.weight.double(), c1.bias.double())
        ref = (xd + res_scale * h).transpose(1, 2)
    assert c3._split is not None and c1._split is not None
    e_exact, e_tc = _err(exact, ref), _err(tc, ref)
    print(f"ResConv1DBlock 1024 rs {res_scale}: exact vs fp64 {e_exact:.1e}, tensor cores vs fp64 {e_tc:.1e}")
    assert e_tc <= max(4e-6, 2 * e_exact)


def _conditioner(out_width, width, down_t, res_scale):
    from jukebox_b200.prior.conditioners import Conditioner
    torch.manual_seed(out_width + width + down_t)
    return Conditioner(input_shape=(2048 if down_t == 2 else 1024,), bins=2048, down_t=down_t, stride_t=2,
                       out_width=out_width, init_scale=1.0, zero_out=False, res_scale=res_scale, width=width, depth=16,
                       m_conv=1.0, dilation_growth_rate=3, dilation_cycle=8, checkpoint_res=1).cuda().eval()


def _conditioner_f64(m, codes):
    from jukebox_b200.vqvae.ops_cl import Conv1d, ConvTranspose1d
    x = m.x_emb.weight.detach().double()[codes].transpose(1, 2)

    def conv(c, x):
        if isinstance(c, ConvTranspose1d):
            return F.conv_transpose1d(x, c.weight.double(), c.bias.double(), stride=2, padding=1)
        return F.conv1d(x, c.weight.double(), c.bias.double(), padding=c.padding, dilation=c.dilation)

    for part in m.cond.model:
        if isinstance(part, Conv1d):
            x = conv(part, x)
            continue
        res, up = part[0], part[1]
        for blk in (res.blocks if res.checkpoint_res == 1 else res.model):
            c3, c1 = blk.model[1], blk.model[3]
            x = x + blk.res_scale * conv(c1, F.relu(conv(c3, F.relu(x))))
        x = conv(up, x)
    x = x.transpose(1, 2)
    return F.layer_norm(x, (m.width,), m.ln.weight.double(), m.ln.bias.double(), m.ln.eps)


@pytest.mark.parametrize("geometry", ["upsampler_level_0", "upsampler_level_1", "small_upsampler"])
def test_conditioner_routes_agree(geometry):
    """the whole Conditioner: tensor-core route vs exact route vs float64, after the LayerNorm"""
    from jukebox_b200.vqvae.resnet import use_tensor_cores
    if geometry == "small_upsampler":
        m = _conditioner(1024, 512, 3, False)
    else:
        m = _conditioner(1920, 1024, 2, geometry == "upsampler_level_1")
    codes = torch.randint(0, 2048, (2, m.x_shape[0]), device="cuda")
    with torch.no_grad():
        tc = m(codes)
        use_tensor_cores(m, False)
        exact = m(codes)
        use_tensor_cores(m, True)
        ref = _conditioner_f64(m, codes)
    e_tc, e_exact, e_routes = _err(tc, ref), _err(exact, ref), _err(tc, exact.double())
    print(f"Conditioner {geometry}: tensor cores vs fp64 {e_tc:.1e}, exact vs fp64 {e_exact:.1e}, routes {e_routes:.1e}")
    assert e_tc <= 2e-5 and e_routes <= 2e-5


@pytest.mark.parametrize("kind,dil,ci,co", [("k3", 27, 1024, 1920), ("up", 1, 1024, 512), ("k3", 2187, 192, 320)])
def test_clip_alone_equals_clip_in_batch(kind, dil, ci, co):
    torch.manual_seed(11)
    m = _module(kind, dil, ci, co)
    m.tensor_cores = True
    x = torch.randn(4, 1000, ci, device="cuda")
    with torch.no_grad():
        batch = m(x)
        for i in range(4):
            alone = m(x[i:i + 1].clone())
            assert torch.equal(alone[0], batch[i]), (kind, i)


@pytest.mark.parametrize("kind,dil,ci,co", [("k3", 27, 1024, 1920), ("up", 1, 1024, 1024)])
def test_tensor_cores_off_is_the_exact_kernel(kind, dil, ci, co):
    """tensor_cores = False is bitwise jk_conv1d_cl's exact kernel (which ignores the flag for wide shapes)"""
    import ctypes as C
    from jukebox_b200 import _lib
    from jukebox_b200.vqvae.ops_cl import _conv
    torch.manual_seed(5)
    m = _module(kind, dil, ci, co)
    x = torch.randn(2, 1000, ci, device="cuda")
    with torch.no_grad():
        off = m(x)
        w, b = m.packed()
        if kind == "up":
            phases = m._phases
            ref = torch.empty_like(off)
            for p, taps in ((0, [0, -1]), (1, [1, 0])):
                _conv(x, phases[p], b, 1000, co, taps, out=ref, out_stride=2, out_offset=p, tensor_cores=True)
        else:
            ref = _conv(x, w, b, 1000, co, m.taps, tensor_cores=True)
    assert m._split is None
    assert torch.equal(off, ref)
