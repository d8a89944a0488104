"""Development aid: summarise the per-phase timeline k_step_resident dumps with PBD_B200_TRACE=<file> (globaltimer, ns).
Record per (phase, CTA): [0] phase start, [1] X items done, [2] other items done + cluster arrive issued, [3] cluster wait returned,
[4] X wait returned (0 where the CTA has no X items in the phase: the integration phase, or no X item of its own in the colour).
Stamps 0, 2 and 3 are written by thread 0 (it runs shared-memory items, "R items"), stamps 1 and 4 by the first X thread: the two run
concurrently, so the R side of a phase is [2] - [0], and [2] - [1] is how long the R side runs on after the X warps have published."""
import sys
import numpy as np

SLOTS = 5
path, ctas = sys.argv[1], int(sys.argv[2])
a = np.fromfile(path, dtype=np.uint64).reshape(-1, ctas, SLOTS).astype(np.float64)
valid = (a[:, :, 0] > 0).all(axis=1) & (a[:, :, 3] > 0).all(axis=1)
a = a[valid]
print("phases recorded:", len(a), "CTAs:", ctas)
t0 = a[0, :, 0].min()
x = a[:, :, 1] - a[:, :, 0]; r = a[:, :, 2] - a[:, :, 0]; tail = a[:, :, 2] - a[:, :, 1]; w = a[:, :, 3] - a[:, :, 2]
has_xw = a[:, :, 4] > 0
xw = np.where(has_xw, a[:, :, 4] - a[:, :, 0], np.nan)  # phase start -> X wait returned
period = np.diff(a[:, :, 0].min(axis=1))
print("phase period (first CTA start to next phase's first CTA start): mean %.0f ns, median %.0f, p95 %.0f" % (period.mean(), np.median(period), np.percentile(period, 95)))
for name, v in (("X items (incl. wait)", x), ("R items (thread 0)", r), ("R tail after X publish", tail), ("cluster wait", w)):
    print("%-22s per CTA: mean %.0f ns, median %.0f, p95 %.0f, max-over-CTAs mean %.0f" % (name, v.mean(), np.median(v), np.percentile(v, 95), v.max(axis=1).mean()))
if has_xw.any():
    v = xw[has_xw]
    print("%-22s per CTA: mean %.0f ns, median %.0f, p95 %.0f, max-over-CTAs mean %.0f (%d of %d CTA-phases wait)" % (
        "X wait", v.mean(), np.median(v), np.percentile(v, 95), np.nanmax(xw[has_xw.any(axis=1)], axis=1).mean(), has_xw.sum(), has_xw.size))
    print("%-22s per CTA: mean %.0f ns, median %.0f" % ("X items after wait", np.nanmean(x - xw), np.nanmedian(x - xw)))
skew = a[:, :, 0].max(axis=1) - a[:, :, 0].min(axis=1)
print("start skew across CTAs: mean %.0f ns, median %.0f, p95 %.0f" % (skew.mean(), np.median(skew), np.percentile(skew, 95)))
n = min(12, len(a))
print("first phases (us since start; per phase: start min..max | work max | X wait mean..max | cluster wait min..max):")
for p in range(n):
    xwp = xw[p][has_xw[p]]
    xws = "%.2f..%.2f" % (xwp.mean() / 1e3, xwp.max() / 1e3) if len(xwp) else "-"
    print("  %3d: start %.2f..%.2f | X %.2f R %.2f (max) | X wait %s | wait %.2f..%.2f" % (p, (a[p, :, 0].min() - t0) / 1e3, (a[p, :, 0].max() - t0) / 1e3, x[p].max() / 1e3,
                                                                                    r[p].max() / 1e3, xws, w[p].min() / 1e3, w[p].max() / 1e3))
