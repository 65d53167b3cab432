"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: per-kernel time of the LAST level-0 block
(single lane), plus the launch sequence of the solver kernels.  ncu serialises launches and runs them cold-cache, so the
SHARES are meaningful, not the absolutes."""
import collections
import csv
import sys

rows = list(csv.reader(open(sys.argv[1])))
hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
hdr = rows[hi]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
data = [(r[ki].split("(")[0], float(r[vi].replace(",", ""))) for r in rows[hi + 1:] if len(r) > vi]
idx = [i for i, (k, v) in enumerate(data) if "bed_relayout" in k]
blk = data[idx[-1]:]
if len(idx) >= 2 and not any('l0_std_apply' in k for k, v in blk):      # capture ended inside the last block: take the one before
    blk = data[idx[-2]:idx[-1]]
tot = collections.OrderedDict()
for k, v in blk:
    tot.setdefault(k, [0.0, 0])
    tot[k][0] += v / 1000
    tot[k][1] += 1
total = sum(t for t, n in tot.values())
print("# %s: last level-0 block of the run (us, launches, share)" % sys.argv[1])
for k, (t, n) in tot.items():
    print("%-46s %9.1f  x%-3d %5.1f%%" % (k.replace("rg::", "").replace("void ", "")[:46], t, n, 100 * t / total))
print("%-46s %9.1f" % ("sum", total))
print("# solver launch sequence (us):")
print(" ".join("%s:%.0f" % (k.replace("rg::", "").replace("void ", "").replace("_kernel", "")[:14], v / 1000)
               for k, v in blk if any(s in k for s in ("tf32", "potrf", "mx_", "chol_"))))
