"""Device time of the fused bottleneck tail vs the two-kernel path (CUDA events, back-to-back launches), and of the fp16-split
('exact' math) bottleneck at the cfg2 shapes: conv1 writing fp32 + the tail splitting it on the SM (fused_h3) against conv1
writing split pairs + the tail reading them (fused_h3_split).  The split rows also report the L2->SM bytes of the tail over its
time (A slabs of 9 (dy, dz) pairs x 1.25 bricks per K slice + the three x-taps' weight tiles per stage + W3, per brick)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-sis_b200"))
import torch
from lib import _sis3d as S
DEV = torch.device("cuda", 0)


def timed(f, n=200):
    for _ in range(20): f()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): f()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / n


print(torch.cuda.get_device_name(0))
for cin, cmid, cout, dims in [(32, 32, 64, (48, 24, 48)), (32, 32, 32, (48, 24, 48)), (64, 64, 128, (24, 12, 24)), (32, 32, 64, (24, 12, 24))]:
    x = torch.randn(*dims, cin, device=DEV); r = torch.randn(*dims, cout, device=DEV)
    w2 = torch.randn(cmid, 27 * cin, device=DEV) * 0.05; w3 = torch.randn(cout, cmid, device=DEV) * 0.1
    mid = torch.empty(*dims, cmid, device=DEV); out = torch.empty(*dims, cout, device=DEV)
    st = S.stream()
    def fused():
        S.check(S.lib.sis3d_conv3d_k3_tc_fused(S.ptr(x), S.ptr(w2), None, S.ptr(w3), None, S.ptr(r), cout, 0, S.ptr(out), cout, 0, *dims, cin, cmid, cout, 1, st))
    def two():
        S.check(S.lib.sis3d_conv3d_k3_tc(S.ptr(x), S.ptr(w2), None, None, 0, 0, S.ptr(mid), cmid, 0, *dims, cin, cmid, 3, None, 0, 1, st))
        S.check(S.lib.sis3d_conv3d_k3_tc(S.ptr(mid), S.ptr(w3), None, S.ptr(r), cout, 0, S.ptr(out), cout, 0, *dims, cmid, cout, 1, None, 0, 1, st))
    for name, f in (("fused", fused), ("two", two)):
        print(cin, cmid, cout, dims, name, "%.2f us" % timed(f))

# 'exact' math bottleneck: block input xin (cout channels) -> conv1 (1x1, cout -> cin) -> tail (cin -> cmid -> cout, + xin)
for cin, cmid, cout, dims in [(32, 32, 32, (48, 24, 48)), (32, 32, 64, (48, 24, 48)), (64, 64, 128, (24, 12, 24))]:
    xin = torch.randn(*dims, cout, device=DEV)
    w1 = torch.randn(cin, cout, 1, 1, 1, device=DEV) * 0.1; b1 = torch.randn(cin, device=DEV)
    w2 = torch.randn(cmid, cin, 3, 3, 3, device=DEV) * 0.05; w3 = torch.randn(cout, cmid, 1, 1, 1, device=DEV) * 0.1
    b2, b3 = torch.randn(cmid, device=DEV), torch.randn(cout, device=DEV)
    wh = []
    for w in (w1, w2, w3):
        h = torch.empty(2 * w.shape[0], w[0].numel(), dtype=torch.float16, device=DEV)
        S.check(S.lib.sis3d_pack_conv_weight_tc_h3(S.ptr(w), w.shape[0], w.shape[1], w.shape[2], S.ptr(h), S.stream()))
        wh.append(h)
    y = torch.empty(*dims, cin, device=DEV); ys = torch.empty(*dims, 2 * cin, dtype=torch.float16, device=DEV)
    out = torch.empty(*dims, cout, device=DEV)
    st = S.stream()
    conv1 = lambda: S.check(S.lib.sis3d_conv3d_k3_tc_h3(S.ptr(xin), S.ptr(wh[0]), S.ptr(b1), None, 0, 0, S.ptr(y), cin, 0, *dims, cout, cin, 1, 1, st))  # noqa: E731
    conv1s = lambda: S.check(S.lib.sis3d_conv3d_k1_tc_h3_split(S.ptr(xin), S.ptr(wh[0]), S.ptr(b1), S.ptr(ys), *dims, cout, cin, 1, st))  # noqa: E731
    tail = lambda: S.check(S.lib.sis3d_conv3d_k3_tc_fused_h3(S.ptr(y), S.ptr(wh[1]), S.ptr(b2), S.ptr(wh[2]), S.ptr(b3), S.ptr(xin), cout, 0, S.ptr(out), cout, 0, *dims, cin, cmid, cout, 1, st))  # noqa: E731
    tails = lambda: S.check(S.lib.sis3d_conv3d_k3_tc_fused_h3_split(S.ptr(ys), S.ptr(wh[1]), S.ptr(b2), S.ptr(wh[2]), S.ptr(b3), S.ptr(xin), cout, 0, S.ptr(out), cout, 0, *dims, cin, cmid, cout, 1, st))  # noqa: E731
    bricks = -(-dims[0] // 8) * -(-dims[1] // 2) * -(-dims[2] // 8)
    tail_bytes = bricks * (cin // 32) * 9 * (160 * 128 + 3 * cmid * 128) + bricks * cout * cmid * 4
    t = {k: timed(f) for k, f in (("conv1 fp32", conv1), ("conv1 split", conv1s), ("tail fused_h3", tail), ("tail fused_h3_split", tails))}
    for k, v in t.items():
        extra = f"  L2->SM {tail_bytes / (v * 1e-6) / 1e12:.2f} TB/s ({tail_bytes / 1e6:.0f} MB)" if k.startswith("tail") else ""
        print(f"h3 bottleneck {cin}/{cmid}/{cout} {dims} {k}: {v:.2f} us{extra}")
    print(f"h3 bottleneck {cin}/{cmid}/{cout} {dims} conv1 + tail: {t['conv1 fp32'] + t['tail fused_h3']:.2f} -> "
          f"{t['conv1 split'] + t['tail fused_h3_split']:.2f} us")
