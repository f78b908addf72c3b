"""The persistent, warp-specialized wgmma GEMM (gemm_tc_kernel: every tensor-core GEMM with more than one M tile, a
batch, or a head-major output) against a float64 torch product of the same SB16 values, on the operand layouts and
epilogues the encoder and the cross-K/V projection use."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _eng():
    from whisper_timestamped.engine import CudaEngine
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = torch.device("cuda:0"), 0, 0
    return eng


def _sb(x):
    from whisper_timestamped.model import SB16
    return SB16.from_f32(x.contiguous())


def _ref(A):
    """float64 values of an SB16 operand (the kernel's input, exactly)."""
    return A.to_f32().double()


def _check(got, ref, tol):
    scale = max(1.0, ref.abs().max().item())
    err = (got.double() - ref).abs().max().item()
    assert err <= tol * scale, (err, scale)


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_more_tiles_than_sms_ragged_tails():
    """Ragged M/N/K tails, several tiles per CTA (both consumers, several ring laps), GELU + residual, float32 and SB16
    outputs at once."""
    from whisper_timestamped.model import SB16
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(21)
    for (M, N, K) in [(2900, 1900, 1288), (1500, 5120, 72), (24000 // 8, 1280, 5120 + 8)]:
        assert ((M + 127) // 128) * ((N + 127) // 128) > _n_sm()
        a = torch.randn(M, K, generator=g).to(dev)
        b = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        res = torch.randn(M, N, generator=g).to(dev)
        A, Bm = _sb(a), _sb(b)
        out = torch.full((M, N), 7.0, device=dev)
        osb = SB16(M, N, dev)
        eng.gemm(A, Bm, M, N, K, bias=bias, act=1, residual=res, ldr=N, out_f32=out, ldc=N, out_sb=osb)
        torch.cuda.synchronize()
        ref = torch.nn.functional.gelu(_ref(A) @ _ref(Bm).T + bias.double()) + res.double()
        _check(out, ref, 2e-4)
        _check(osb.to_f32(), ref, 3e-4)


def test_fewer_tiles_than_sms():
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(22)
    for (M, N, K) in [(129, 100, 64), (256, 256, 200), (1000, 300, 136)]:
        assert ((M + 127) // 128) * ((N + 127) // 128) < _n_sm()
        a = torch.randn(M, K, generator=g).to(dev)
        b = torch.randn(N, K, generator=g).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        A, Bm = _sb(a), _sb(b)
        out = torch.zeros(M, N, device=dev)
        eng.gemm(A, Bm, M, N, K, bias=bias, out_f32=out, ldc=N)
        torch.cuda.synchronize()
        _check(out, _ref(A) @ _ref(Bm).T + bias.double(), 2e-4)


def test_batched_with_shared_operands():
    """batch_outer x batch_inner; A varies with both levels, B is shared over the inner level (zero stride) and the
    SB16 output lands in a strided batch layout."""
    from whisper_timestamped.model import SB16
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(23)
    BO, BI, M, N, K = 3, 4, 300, 200, 136
    a = torch.randn(BO * BI * M, K, generator=g).to(dev)
    b = torch.randn(BO * N, K, generator=g).to(dev)
    A, Bm = _sb(a), _sb(b)
    osb = SB16(BO * BI * M, N, dev)
    eng.gemm(A, Bm, M, N, K, batch=(BO, BI), a_b=(BI * M * K, M * K), b_b=(N * K, 0), alpha=0.5,
             out_sb=osb, o_b=(BI * M * N, M * N))
    torch.cuda.synchronize()
    ra, rb = _ref(A).view(BO, BI, M, K), _ref(Bm).view(BO, 1, N, K)
    ref = 0.5 * (ra @ rb.transpose(-1, -2))
    _check(osb.to_f32().view(BO, BI, M, N), ref, 3e-4)


def test_bias_on_m_swapped_operands():
    """V^T per window: A = the shared weight [D, D], B = the window's activations, bias along M, SB16 output with a
    padded row pitch."""
    from whisper_timestamped.model import SB16
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(24)
    B, D, T, LDO = 3, 384, 1500, 1504
    w = (torch.randn(D, D, generator=g) / D ** 0.5).to(dev)
    h = torch.randn(B * T, D, generator=g).to(dev)
    bias = torch.randn(D, generator=g).to(dev)
    W, Hs = _sb(w), _sb(h)
    vt = SB16(B * D, LDO, dev)
    eng.gemm(W, Hs, D, T, D, batch=(B, 1), b_b=(T * D, 0), bias=bias, bias_on_m=True, out_sb=vt, ldo=LDO,
             o_b=(D * LDO, 0))
    torch.cuda.synchronize()
    ref = _ref(W) @ _ref(Hs).view(B, T, D).transpose(-1, -2) + bias.double()[:, None]
    _check(vt.to_f32().view(B, D, LDO)[:, :, :T], ref, 3e-4)
    assert vt.to_f32().view(B, D, LDO)[:, :, T:].abs().max().item() == 0.0


def test_inplace_residual():
    """x += A W^T + b with out_f32 == residual (the encoder's out-projection and fc2)."""
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(25)
    for (M, N, K) in [(3000, 640, 1280), (1500, 384, 1536)]:
        a = torch.randn(M, K, generator=g).to(dev)
        b = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        x = torch.randn(M, N, generator=g).to(dev)
        A, Bm = _sb(a), _sb(b)
        ref = x.double() + _ref(A) @ _ref(Bm).T + bias.double()
        eng.gemm(A, Bm, M, N, K, bias=bias, residual=x, ldr=N, out_f32=x, ldc=N)
        torch.cuda.synchronize()
        _check(x, ref, 2e-4)


def test_head_major_scatter():
    """Cross-K/V projection: output column n of row t of window b goes to [b, n // 64, t, n % 64]."""
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(26)
    B, T, D, H = 2, 1500, 384, 6
    xa = torch.randn(B * T, D, generator=g).to(dev)
    w = (torch.randn(D, D, generator=g) / D ** 0.5).to(dev)
    bias = torch.randn(D, generator=g).to(dev)
    X, W = _sb(xa), _sb(w)
    out = torch.full((B, H, T, 64), 7.0, device=dev)
    eng.gemm(X, W, T, D, D, batch=(B, 1), a_b=(T * D, 0), bias=bias, out_f32=out, ldc=64, c_b=(H * T * 64, 0),
             head_dim=64, head_stride=T * 64)
    torch.cuda.synchronize()
    ref = (_ref(X).view(B, T, D) @ _ref(W).T + bias.double()).view(B, T, H, 64).permute(0, 2, 1, 3)
    _check(out, ref, 2e-4)


def test_conv_overlapping_rows():
    """conv1 / conv2 as GEMMs whose A rows overlap (lda < K): row t of window b reads padded input rows
    s*t .. s*t + 2 (K = 3C), GELU, SB16 output shifted by one row."""
    from whisper_timestamped.model import SB16
    eng = _eng()
    dev = eng.dev
    g = torch.Generator(device="cpu").manual_seed(27)
    B, C, D = 3, 128, 384
    for (T_in, stride, T_out) in [(3000, 1, 3000), (3000, 2, 1500)]:
        rows = T_in + 3 - stride                       # 3002 padded rows for stride 1, 3001 for stride 2
        x = torch.randn(B * rows, C, generator=g).to(dev)
        w = (torch.randn(D, 3 * C, generator=g) / (3 * C) ** 0.5).to(dev)
        bias = torch.randn(D, generator=g).to(dev)
        X, W = _sb(x), _sb(w)
        out = SB16(B * (T_out + 1), D, dev)
        eng.gemm(X, W, T_out, D, 3 * C, lda=stride * C, batch=(B, 1), a_b=(rows * C, 0), bias=bias, act=1,
                 out_sb=out, ldo=D, o_b=((T_out + 1) * D, 0), o_off=D)
        torch.cuda.synchronize()
        xv = _ref(X).view(B, rows, C)
        unf = xv.unfold(1, 3, stride).permute(0, 1, 3, 2).reshape(B, T_out, 3 * C)
        ref = torch.nn.functional.gelu(unf @ _ref(W).T + bias.double())
        got = out.to_f32().view(B, T_out + 1, D)
        _check(got[:, 1:], ref, 3e-4)
        assert got[:, 0].abs().max().item() == 0.0
