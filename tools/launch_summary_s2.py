"""Summarise the `ncu --metrics gpu__time_duration.sum --csv` launch list of tools/step2_probe.py: the kernels of the last
quantitative-trait block on .bed rows and of the last binary-trait block on 8-bit dosages (us, launches, share).  ncu
serialises launches and runs them cold-cache: the SHARES are meaningful, not the absolutes."""
import collections
import csv
import sys

rows = list(csv.reader(open(sys.argv[1])))
hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
hdr = rows[hi]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
data = [(r[ki].split("(")[0], float(r[vi].replace(",", ""))) for r in rows[hi + 1:] if len(r) > vi]


def show(title, blk):
    tot = collections.OrderedDict()
    for k, v in blk:
        tot.setdefault(k, [0.0, 0])
        tot[k][0] += v / 1000
        tot[k][1] += 1
    total = sum(t for t, n in tot.values()) or 1.0
    print("# %s (us, launches, share)" % title)
    for k, (t, n) in tot.items():
        print("%-46s %9.1f  x%-3d %5.1f%%" % (k.replace("rg::", "").replace("void ", "")[:46], t, n, 100 * t / total))
    print("%-46s %9.1f" % ("sum", total))


bed = [i for i, (k, v) in enumerate(data) if "bed_relayout" in k]
dos = [i for i, (k, v) in enumerate(data) if "dosage_relayout" in k]
print("# %s" % sys.argv[1])
if bed:
    end = dos[0] if dos and dos[0] > bed[-1] else len(data)
    fin = [i for i in range(bed[-1], end) if "s2_finalize" in data[i][0]]      # what follows is the probe setting up the next handle
    end = fin[-1] + 1 if fin else end
    show("last QT block: 1000 .bed variants, N = 100k, 10 traits", data[bed[-1]:end])
if dos:
    show("last BT block: 400 variants of 8-bit dosages, N = 100k, 1 binary trait", data[dos[-1]:])
