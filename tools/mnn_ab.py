#!/usr/bin/env python
"""A/B timing of the xfeat_mnn_match implementations on the BASELINE config-2 matching load (64 pairs x 4096 x 4096), in one
process.  python tools/mnn_ab.py  -> one JSON line: ms per call for impl 1 (wgmma, one GEMM per pair, default), 2 (wgmma,
persistent, one GEMM per direction), 3 (one CTA per row block and direction) and 0 (fp32 SIMT), and whether each returns
what impl 1 returns."""
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from accelerated_features_b200 import XFeat  # noqa: E402

xf = XFeat(top_k=4096)
g = torch.Generator().manual_seed(0)
B, N = 64, 4096
f1 = F.normalize(torch.randn(B, N, 64, generator=g), dim=-1).cuda()
f2 = F.normalize(torch.randn(B, N, 64, generator=g), dim=-1).cuda()
out = {}
ref = None
for impl in (1, 2, 3, 0):
    xf._lib.xfeat_set_mnn_impl(impl)
    for _ in range(3):
        r = xf._mnn_device(f1, None, N, N * 64, f2, None, N, N * 64, B, -1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        r = xf._mnn_device(f1, None, N, N * 64, f2, None, N, N * 64, B, -1)
    e1.record()
    torch.cuda.synchronize()
    out[f"impl{impl}_ms"] = e0.elapsed_time(e1) / 10
    print(f"impl {impl}: {out[f'impl{impl}_ms']:.3f} ms", file=sys.stderr, flush=True)
    cnt = r[2].clone()
    if ref is None:
        ref = (r[0].clone(), r[1].clone(), cnt)
    else:
        out[f"impl{impl}_equal_impl1"] = bool(torch.equal(cnt, ref[2]) and torch.equal(r[0], ref[0]) and torch.equal(r[1], ref[1]))
xf._lib.xfeat_set_mnn_impl(1)
print(json.dumps(out))
