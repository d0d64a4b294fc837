"""One layer through the wgmma convs (both forms) and the mma.sync 3xTF32 conv, a few launches each: the target of an
`ncu -k regex:conv5 --set full --import-source on` capture.

    python tools/conv5_probe.py N cin cout ks stride pad dil h w
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops  # noqa: E402

N, cin, cout, ks, S, pad, dil, h, w = (int(a) for a in sys.argv[1:10])
g = torch.Generator().manual_seed(0)
x = torch.randn(N, cin, h, w, generator=g).cuda().contiguous(memory_format=torch.channels_last)
wt = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).cuda()
b = torch.randn(cout, generator=g).cuda()
f3, f5 = ops.pack_conv_filter(wt, 3), ops.pack_conv_filter_tc5(wt)
for _ in range(3):
    ops.conv2d_nhwc(x, f3, b, cout, ks, S, pad, dil, relu=True, precision=3)
    ops.conv2d_tc5(x, f5, b, cout, ks, S, pad, dil, relu=True)
    if S == 1:
        ops.conv2d_tc5(x, ops.pack_conv_filter_tc5h(wt), b, cout, ks, 1, pad, dil, relu=True, halo=True)
torch.cuda.synchronize()
print("ok")

if S == 1 and os.environ.get("C5_TRACE"):
    import json
    from patchmatchnet_b200 import _native
    buf = torch.zeros(256, dtype=torch.int64, device="cuda")
    f5h = ops.pack_conv_filter_tc5h(wt)
    _native.lib().pmb200_debug_conv5h_trace(buf.data_ptr())
    ops.conv2d_tc5(x, f5h, b, cout, ks, 1, pad, dil, relu=True, halo=True)
    torch.cuda.synchronize()
    _native.lib().pmb200_debug_conv5h_trace(None)
    t = buf.cpu().view(4, 16, 4)
    t0 = int(t[t > 0].min())
    rel = torch.where(t > 0, t - t0, torch.full_like(t, -1))
    names = {0: ("producer", ["halo requested"]), 1: ("mma", ["acc free", "planes split", "issued"]),
             2: ("split", ["halo landed", "planes free", "done"]), 3: ("epilogue", ["acc full", "stored"])}
    out = {}
    for r, (name, evs) in names.items():
        out[name] = [{e: int(rel[r, it, k]) for k, e in enumerate(evs)} for it in range(16) if int(t[r, it, 0]) > 0]
    print(json.dumps({"layer": sys.argv[1:10], "clock64_cycles_from_first_event": out}))
