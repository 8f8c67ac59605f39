"""CPU: the routing predicate of the dense GEMM front end (gemm.h gemm_route, through car_op_gemm_route) and the refusals of
gemm(), gemm_f32 and gemm_f32_conv3.  Nothing here touches a device: the pointers are 16-byte-aligned stand-ins that are never
dereferenced, because every call either only routes or is refused before any launch."""
import pytest

from controlar_b200 import _lib
from controlar_b200.engine import gemm_desc, op_gemm_route

WGMMA, WGMMA_CONV3, MMA, MMA_WIN = 0, 1, 2, 3
P = 1 << 20                                             # a 16-byte-aligned stand-in pointer


def plain(**change):
    """A wgmma-eligible plain GEMM: 256 x 128 x 64, bias, all operands aligned."""
    f = dict(A=P, B=P, C=P, M=256, N=128, K=64, lda=64, ldb=64, ldc=128, bias=P)
    return {**f, **change}


def conv(**change):
    """An exact-fit 3x3 convolution: 2 images of 16 x 32 pixels, 64 channels."""
    f = dict(A=P, B=P, C=P, M=2 * 16 * 32, N=64, K=9 * 64, ldb=9 * 64, ldc=64, amode=1, Hs=16, Ws=32, Cin=64, Ho=16, Wo=32)
    return {**f, **change}


def win(**change):
    """A 3 x 3 / stride 2 window over a 17 x 17 source into an 8 x 8 map."""
    f = dict(A=P, B=P, C=P, M=2 * 8 * 8, N=24, K=9 * 24, ldb=9 * 24, ldc=24, amode=3, Hs=17, Ws=17, Cin=24, Ho=8, Wo=8, kh=3, kw=3,
             ws=2, bias_f=P, out_mode=1, osy=1, osx=1, oH=8, oW=8)
    return {**f, **change}


ROUTES = [
    ("plain", plain(), 1, WGMMA),
    ("gelu_tanh", plain(act=1), 1, WGMMA),
    ("gelu_erf", plain(act=2), 1, WGMMA),
    ("scale_resid", plain(scale=P, resid=P, ldr=128), 1, WGMMA),
    ("alpha_zero_means_one", plain(alpha=0.0), 1, WGMMA),
    ("relu", plain(act=3), 1, MMA),
    ("alpha", plain(alpha=0.125), 1, MMA),
    ("bias_along_m", plain(bias_along_m=1), 1, MMA),
    ("bias_f", plain(bias_f=P), 1, MMA),
    ("resid_f", plain(resid_f=P, ldr=128), 1, MMA),
    ("out_mode1", plain(out_mode=1), 1, MMA),
    ("out_mode2", plain(out_mode=2, ldc=0, Ho=16, Wo=16), 1, MMA),
    ("batch", plain(sA=256 * 64, sB=0, sC=256 * 128), 3, MMA),
    ("n_tail", plain(N=100, ldc=104), 1, MMA),
    ("n_257", plain(N=257, ldc=264), 1, MMA),
    ("ldc_odd", plain(ldc=130), 1, MMA),
    ("c_misaligned", plain(C=P + 2), 1, MMA),
    ("resid_misaligned", plain(resid=P + 2, ldr=128), 1, MMA),
    ("ldr_odd", plain(resid=P, ldr=129), 1, MMA),
    ("m_one", plain(M=1), 1, WGMMA),
    ("k8", plain(K=8, lda=8, ldb=8), 1, WGMMA),
    ("conv_exact_fit", conv(), 1, WGMMA_CONV3),
    ("conv_min_map", conv(M=8 * 16, Hs=8, Ws=16, Ho=8, Wo=16), 1, WGMMA_CONV3),
    ("conv_ups", conv(ups=1, Ho=32, Wo=64, M=2 * 32 * 64), 1, MMA),
    ("conv_cin_24", conv(Cin=24, K=9 * 24, ldb=9 * 24), 1, MMA),
    ("conv_hs_small", conv(Hs=7, Ho=7, M=2 * 7 * 32), 1, MMA),
    ("conv_ws_small", conv(Ws=15, Wo=15, M=2 * 16 * 15), 1, MMA),
    ("conv_relu", conv(act=3), 1, MMA),
    ("conv_nchw", conv(out_mode=2, ldc=0, bias_f=P), 1, MMA),
    ("conv_s2", conv(amode=2, Ho=8, Wo=16, M=2 * 8 * 16), 1, MMA),
    ("window", win(), 1, MMA_WIN),
    ("window_pixel_map", win(osy=2, osx=2, oay=1, oax=1, oH=17, oW=17), 1, MMA_WIN),
    ("empty_m", plain(M=0), 1, WGMMA),
]


@pytest.mark.parametrize("name,fields,batch,route", ROUTES, ids=[r[0] for r in ROUTES])
def test_route_table(name, fields, batch, route):
    got = op_gemm_route(gemm_desc(**fields), batch)
    assert got == route, (name, got, _lib.lib().car_last_error())


REFUSED = [
    ("null_a", plain(A=None), 1),
    ("null_b", plain(B=None), 1),
    ("null_c", plain(C=None), 1),
    ("negative_m", plain(M=-1), 1),
    ("k_zero", plain(K=0, lda=8, ldb=8), 1),
    ("k_negative", plain(K=-8), 1),
    ("k_not_8", plain(K=60), 1),
    ("lda_not_8", plain(lda=68), 1),
    ("lda_lt_k", plain(lda=56), 1),
    ("ldb_not_8", plain(ldb=68), 1),
    ("ldb_lt_k", plain(ldb=56), 1),
    ("ldc_lt_n", plain(ldc=120), 1),
    ("a_misaligned", plain(A=P + 8), 1),
    ("b_misaligned", plain(B=P + 2), 1),
    ("batch_zero", plain(), 0),
    ("batch_huge", plain(), 65536),
    ("batch_sa_not_8", plain(sA=256 * 64 + 4), 2),
    ("batch_sb_not_8", plain(sB=4), 2),
    ("amode", plain(amode=4), 1),
    ("act", plain(act=4), 1),
    ("out_mode", plain(out_mode=3), 1),
    ("bias_along_m_without_bias", plain(bias=None, bias_along_m=1), 1),
    ("resid_ldr_lt_n", plain(resid=P, ldr=64), 1),
    ("resid_f_ldr_lt_n", plain(resid_f=P, ldr=64, out_mode=1), 1),
    ("scale_fp32_out", plain(scale=P, out_mode=1), 1),
    ("resid_fp32_out", plain(resid=P, ldr=128, out_mode=1), 1),
    ("gelu_fp32_out", plain(act=1, out_mode=1), 1),
    ("gelu_erf_nchw", conv(act=2, out_mode=2, ldc=0), 1),
    ("nchw_batch", conv(out_mode=2, ldc=0, sA=0, sB=0), 2),
    ("nchw_ldc", conv(out_mode=2, ldc=64), 1),
    ("nchw_m_not_image", plain(out_mode=2, ldc=0, Ho=15, Wo=15), 1),
    ("conv_cin_not_8", conv(Cin=20, K=180, ldb=184), 1),
    ("conv_k_not_9cin", conv(K=8 * 64), 1),
    ("conv_m_not_image", conv(M=2 * 16 * 32 + 1), 1),
    ("conv_zero_source", conv(Hs=0), 1),
    ("conv_ups_2", conv(ups=2), 1),
    ("conv_s2_ups", conv(amode=2, ups=1, Ho=16, Wo=32), 1),
    ("window_without_bias_f", win(bias_f=None), 1),
    ("window_bf16_out", win(out_mode=0), 1),
    ("window_nchw", win(out_mode=2, ldc=0), 1),
    ("window_batch", win(), 2),
    ("window_alpha", win(alpha=0.5), 1),
    ("window_bias", win(bias=P), 1),
    ("window_act", win(act=3), 1),
    ("window_gelu", win(act=1), 1),
    ("window_scale", win(scale=P), 1),
    ("window_resid", win(resid=P, ldr=24), 1),
    ("window_resid_f", win(resid_f=P, ldr=24), 1),
    ("window_k", win(K=8 * 24), 1),
    ("window_reads_past_source", win(Hs=16), 1),
    ("window_reads_past_source_w", win(Ws=16), 1),
    ("window_kernel_zero", win(kh=0, K=0), 1),
    ("window_stride_zero", win(ws=0), 1),
    ("window_map_outside", win(oH=7), 1),
    ("window_map_outside_w", win(osx=2, oW=14), 1),
    ("window_map_offset_negative", win(oay=-1), 1),
    ("window_ldc_lt_n", win(ldc=16), 1),
    ("window_cin_not_8", win(kh=2, kw=2, Cin=2, K=8, ldb=8), 1),
]


@pytest.mark.parametrize("name,fields,batch", REFUSED, ids=[r[0] for r in REFUSED])
def test_gemm_refusals(name, fields, batch):
    l = _lib.lib()
    d = gemm_desc(**fields)
    rc = op_gemm_route(d, batch)
    assert rc < 0, (name, rc)
    assert b"gemm_route" in l.car_last_error(), name
    # gemm() refuses the same descriptor before it launches anything (the stand-in pointers are never dereferenced)
    assert l.car_op_gemm(d, batch, None) == rc, name


def test_null_descriptor_is_refused():
    l = _lib.lib()
    assert l.car_op_gemm_route(None, 1) < 0 and l.car_last_error()
    assert l.car_op_gemm(None, 1, None) < 0 and l.car_last_error()


F32 = dict(A=P, B=P, M=100, N=24, K=64, bias=P, resid=P, out=P, ldc=24)
F32_REFUSED = [dict(A=None), dict(B=None), dict(out=None), dict(M=-1), dict(N=0), dict(N=20, ldc=20), dict(K=0), dict(K=60),
               dict(ldc=16), dict(ldc=25), dict(A=P + 8), dict(B=P + 4), dict(out=P + 4), dict(resid=P + 4)]


@pytest.mark.parametrize("change", F32_REFUSED, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_gemm_f32_refusals(change):
    l = _lib.lib()
    a = {**F32, **change}
    rc = l.car_op_gemm_f32(a["A"], a["B"], a["M"], a["N"], a["K"], a["bias"], a["resid"], a["out"], a["ldc"], None)
    assert rc < 0, change
    assert b"gemm_f32" in l.car_last_error(), change


CONV3 = dict(src=P, fh=24, fw=24, B=P, nimg=2, H=12, W=20, cin=64, N=24, bias=P, resid=P, out=P)
CONV3_REFUSED = [dict(src=None), dict(B=None), dict(out=None), dict(nimg=0), dict(H=0), dict(W=-1), dict(cin=0), dict(cin=32),
                 dict(cin=72), dict(N=0), dict(N=20), dict(fh=11), dict(fw=19), dict(H=4, W=10, fh=4, fw=16), dict(H=4, W=10, fh=8, fw=10),
                 dict(src=P + 8), dict(B=P + 2), dict(out=P + 4), dict(resid=P + 4)]


@pytest.mark.parametrize("change", CONV3_REFUSED, ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_gemm_f32_conv3_refusals(change):
    l = _lib.lib()
    a = {**CONV3, **change}
    rc = l.car_op_gemm_f32_conv3(a["src"], a["fh"], a["fw"], a["B"], a["nimg"], a["H"], a["W"], a["cin"], a["N"], a["bias"], a["resid"],
                                 a["out"], None)
    assert rc < 0, change
    assert b"gemm_f32_conv3" in l.car_last_error(), change
