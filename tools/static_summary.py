"""Static evidence about the built library (no GPU needed): per-kernel registers / stack / static shared memory from
`cuobjdump --dump-resource-usage`, and counts of the SASS mnemonics that show the Hopper paths are in the binary
(HGMMA = wgmma, UTMALDG/UTMASTG = TMA tensor copies, UBLKCP = bulk copy, CREDUX / REDUX = redux.sync, SYNCS = mbarrier,
STAS = st.async).  Usage: python tools/static_summary.py  (prints to stdout)"""
import collections, os, re, subprocess, sys

so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3dssd_b200", "libssd3d.so")
res = subprocess.run(["cuobjdump", "--dump-resource-usage", so], capture_output=True, text=True).stdout.splitlines()
print("# %s (%d bytes)" % (os.path.relpath(so), os.path.getsize(so)))
print("# kernel: registers / stack bytes / static shared bytes   (LOCAL is 0 for every kernel unless listed)")
name = None
for ln in res:
    m = re.search(r"Function (\S+):", ln)
    if m:
        name = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
        name = re.sub(r"\(.*", "", name)
        continue
    m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", ln)
    if m and name:
        extra = "  LOCAL:%s" % m.group(4) if m.group(4) != "0" else ""
        print("%-90s %4s / %3s / %6s%s" % (name, m.group(1), m.group(2), m.group(3), extra))
        name = None
sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
cnt = collections.Counter()
per = collections.defaultdict(collections.Counter)
fn = None
for ln in sass.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        fn = m.group(1)
        continue
    m = re.search(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
    if m:
        op = m.group(1)
        for key in ("HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "CREDUX", "REDUX", "SYNCS", "STAS", "UCGABAR", "ATOMG", "RED"):
            if op.startswith(key):
                cnt[key] += 1
                per[key][fn] += 1
print("\n# SASS mnemonic counts over the whole library")
for k, v in sorted(cnt.items(), key=lambda kv: -kv[1]):
    top = ", ".join("%s x%d" % (re.sub(r"\(.*", "", subprocess.run(["c++filt", f], capture_output=True, text=True).stdout.strip())[:60], c)
                    for f, c in per[k].most_common(3))
    print("%-12s %6d   (most in: %s)" % (k, v, top))
