"""Split-pair activations on the GPU: the fp16-split 1x1 conv that writes [32 hi | 32 lo] halves per 32-channel slice, and the
fused bottleneck tail that reads them.  The split must be the one the tail would have made on the SM, so the tail's result is
bit-identical to the fp32-input entry point."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def S():
    from lib import _sis3d
    return _sis3d


def split_pairs(v):
    """fp32 [..., C] -> fp16 [..., 2 C]: per 32-channel slice 32 hi = fp16(v), then 32 lo = fp16((v - hi) * 2048)."""
    hi = v.half()
    lo = ((v - hi.float()) * 2048.0).half()
    sh = v.shape[:-1] + (v.shape[-1] // 32, 32)
    return torch.stack([hi.reshape(sh), lo.reshape(sh)], -2).reshape(v.shape[:-1] + (2 * v.shape[-1],))


def pack_h3(S, w):
    cout, cin, ks = w.shape[0], w.shape[1], w.shape[2]
    wh3 = torch.empty(2 * cout, ks ** 3 * cin, dtype=torch.float16, device=DEV)
    S.check(S.lib.sis3d_pack_conv_weight_tc_h3(S.ptr(w), cout, cin, ks, S.ptr(wh3), S.stream()))
    return wh3


def conv1x1_case(S, cin, cout, dims, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*dims, cin, generator=g).to(DEV)
    w = (torch.randn(cout, cin, 1, 1, 1, generator=g) / cin ** 0.5).to(DEV)
    b = torch.randn(cout, generator=g).to(DEV)
    wh3 = pack_h3(S, w)
    ys = torch.full(dims + (2 * cout,), 7.0, dtype=torch.float16, device=DEV)
    S.check(S.lib.sis3d_conv3d_k1_tc_h3_split(S.ptr(x), S.ptr(wh3), S.ptr(b), S.ptr(ys), *dims, cin, cout, 1, S.stream()))
    return x, w, b, wh3, ys


@pytest.mark.parametrize("cin,cout,dims", [(32, 32, (48, 24, 48)), (64, 32, (45, 27, 41)), (128, 64, (24, 12, 24)),
                                           (64, 256, (17, 9, 11))])
def test_k1_split_equals_split_of_fp32_output(S, cin, cout, dims):
    """(a) the split-pair output is split_f16x2 of the fp32 output of the same conv, bit for bit (cout = 256: the second N
    block writes its rows at the 2 * n0 split-row offset)."""
    x, _, b, wh3, ys = conv1x1_case(S, cin, cout, dims, cin + cout + dims[0])
    y = torch.empty(dims + (cout,), device=DEV)
    S.check(S.lib.sis3d_conv3d_k3_tc_h3(S.ptr(x), S.ptr(wh3), S.ptr(b), None, 0, 0, S.ptr(y), cout, 0, *dims, cin, cout, 1, 1,
                                        S.stream()))
    torch.cuda.synchronize()
    assert torch.equal(ys.view(torch.int16), split_pairs(y).view(torch.int16))


def test_k1_split_matches_fp32_conv(S):
    """(c) at 48x24x48, hi + lo / 2048 matches the fp64 conv within what 22-bit operands allow: each product carries a
    relative error of about 2^-21 and the output split one of 2^-22, so the error stays below 2^-19 of sum |x| |w| + |b|."""
    cin, cout, dims = 32, 32, (48, 24, 48)
    x, w, b, _, ys = conv1x1_case(S, cin, cout, dims, 5)
    torch.cuda.synchronize()
    p = ys.float().reshape(dims + (cout // 32, 2, 32))
    got = (p[..., 0, :] + p[..., 1, :] / 2048.0).reshape(dims + (cout,)).cpu().double()
    xd, wd, bd = x.cpu().double(), w.cpu().double().reshape(cout, cin), b.cpu().double()
    ref = F.relu(xd @ wd.T + bd)
    scale = xd.abs() @ wd.abs().T + bd.abs()
    err = (got - ref).abs()
    assert bool((err <= scale * 2.0 ** -19).all()), f"max err / scale {(err / scale).max().item():.2e}"


@pytest.mark.parametrize("dims", [(48, 24, 48), (24, 12, 24), (45, 27, 41)])
@pytest.mark.parametrize("cin,cmid,cout", [(32, 32, 32), (32, 32, 64), (64, 64, 128)])
def test_fused_tail_split_input_bit_identical(S, cin, cmid, cout, dims):
    """(b) the tail fed split pairs == sis3d_conv3d_k3_tc_fused_h3 on the fp32 tensor they were split from, bit for bit
    (several bricks per SM at 48x24x48, partial edge bricks at 45x27x41), with a residual and an offset output."""
    g = torch.Generator().manual_seed(cin + cout + dims[2])
    y = F.relu(torch.randn(*dims, cin, generator=g)).to(DEV)
    w2 = (torch.randn(cmid, cin, 3, 3, 3, generator=g) / (27 * cin) ** 0.5).to(DEV)
    w3 = (torch.randn(cout, cmid, 1, 1, 1, generator=g) / cmid ** 0.5).to(DEV)
    b2, b3 = torch.randn(cmid, generator=g).to(DEV), torch.randn(cout, generator=g).to(DEV)
    r = torch.randn(*dims, cout, generator=g).to(DEV)
    w2h, w3h = pack_h3(S, w2), pack_h3(S, w3)
    ys = split_pairs(y).contiguous()
    want = torch.full(dims + (cout + 4,), 7.0, device=DEV)
    got = torch.full(dims + (cout + 4,), 7.0, device=DEV)
    S.check(S.lib.sis3d_conv3d_k3_tc_fused_h3(S.ptr(y), S.ptr(w2h), S.ptr(b2), S.ptr(w3h), S.ptr(b3), S.ptr(r), cout, 0, S.ptr(want),
                                              cout + 4, 4, *dims, cin, cmid, cout, 1, S.stream()))
    S.check(S.lib.sis3d_conv3d_k3_tc_fused_h3_split(S.ptr(ys), S.ptr(w2h), S.ptr(b2), S.ptr(w3h), S.ptr(b3), S.ptr(r), cout, 0,
                                                    S.ptr(got), cout + 4, 4, *dims, cin, cmid, cout, 1, S.stream()))
    torch.cuda.synchronize()
    assert torch.all(got[..., :4] == 7.0)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    ref = F.relu(F.conv3d(F.relu(F.conv3d(y.permute(3, 0, 1, 2)[None].double(), w2.double(), b2.double(), padding=1)),
                          w3.double(), b3.double())[0].permute(1, 2, 3, 0) + r.double())
    assert (got[..., 4:].double() - ref).abs().max().item() < 1e-4
