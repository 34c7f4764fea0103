#!/usr/bin/env python
"""Where a stage of the tensor SYRK (syrk_tc_kernel) spends its clocks, by role (BALM_TC_TRACE=1): the benchmark's C3
scene (500 poses x 100 000 plane voxels, tensor path), a few evaluations, then the trace of the last SYRK launch.
Prints clocks per 64-row stage of a 128 x 64 half tile (a whole-tile stage counts as two; mean over the CTAs, and over
the busiest CTA) of every category of balm_debug_tc_trace, the stage count and the SM clock derived from the globaltimer
pair. BALM_TC_TILE=half|full in the environment forces the item shape.
Usage: python scripts/tc_trace.py [N_POSES [N_VOXELS]]"""
import ctypes as C
import json
import os
import sys

import numpy as np

os.environ["BALM_TC_TRACE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import balm_b200  # noqa: E402
from balm_b200 import _lib as L  # noqa: E402

WORDS = 18
ROLES = [("consumer warp 0", 3, ["wait stage full", "warpgroup vote", "wgmma.wait_group", "epilogue", "total"]),
         ("consumer warp 4", 8, ["wait stage full", "warpgroup vote", "wgmma.wait_group", "epilogue", "total"]),
         ("producer", 16, ["wait slot empty", "wait flags"])]
COPY_WORDS = 3

N = int(sys.argv[1]) if len(sys.argv) > 1 else 500
M = int(sys.argv[2]) if len(sys.argv) > 2 else 100000
c = balm_b200.Context(N, 0, balm_b200.PREC_TENSOR)
gt, init = c.synth_virtual(M, 0, 40, 0.01, 2.0, 10)
for _ in range(3):
    c.evaluate(init, want_H=False)
buf = np.zeros(WORDS * 1024, dtype=np.uint64)
L.check(L.lib().balm_debug_tc_trace(c._h, buf.ctypes.data_as(C.c_void_p), len(buf)))
tr = buf.reshape(-1, WORDS).astype(np.int64)
tr = tr[tr[:, 0] > 0]
stages = tr[:, 0]
ghz = tr[:, 7] / np.maximum(tr[:, 2] - tr[:, 1], 1)
busiest = int(np.argmax(stages))
out = {"ctas": len(tr), "stages_total": int(stages.sum()), "stages_max": int(stages.max()),
       "stages_mean": float(stages.mean()), "sm_ghz_mean": float(ghz.mean()),
       "span_us_max": float((tr[:, 2] - tr[:, 1]).max() / 1e3), "digit_planes": c.timings()["digit_planes"]}
print(f"{out['ctas']} CTAs, {out['stages_total']} stages (max {out['stages_max']} per CTA), "
      f"SM clock {out['sm_ghz_mean']:.3f} GHz, longest CTA {out['span_us_max']:.0f} us, S = {out['digit_planes']}")
print(f"{'role':18s} {'category':18s} {'clk/stage mean':>15s} {'busiest CTA':>12s}")
for role, off, cats in ROLES:
    for k, cat in enumerate(cats):
        mean = float((tr[:, off + k] / stages).mean())
        top = float(tr[busiest, off + k] / stages[busiest])
        out[f"{role}/{cat}"] = round(mean, 1)
        print(f"{role:18s} {cat:18s} {mean:15.1f} {top:12.1f}")
cbuf = np.zeros(COPY_WORDS * 1024, dtype=np.uint64)
L.check(L.lib().balm_debug_tc_copy_trace(c._h, cbuf.ctypes.data_as(C.c_void_p), len(cbuf)))
# per CTA: its three copier warps' clocks on their units, of those the clocks waiting on loads, plane tiles copied
ct = cbuf.reshape(-1, COPY_WORDS).astype(np.int64)
ct = ct[ct[:, 2] > 0]
out.update({"copier/plane tiles": int(ct[:, 2].sum()),
            "copier/clk per plane tile": float((ct[:, 0] / ct[:, 2]).mean()),
            "copier/busy share of consumer span": float(ct[:, 0].mean() / 3 / tr[:, 7].mean()),
            "copier/wait share": float(ct[:, 1].sum() / max(ct[:, 0].sum(), 1))})
print(f"copiers: {out['copier/plane tiles']} plane tiles, {out['copier/clk per plane tile']:.0f} clk per tile and warp, "
      f"busy {100 * out['copier/busy share of consumer span']:.1f} % of the consumers' span, "
      f"{100 * out['copier/wait share']:.1f} % of that waiting on loads")
print(json.dumps(out))
c.close()
