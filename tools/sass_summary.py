"""cuobjdump -sass of libc2m_sm100.so -> per-kernel counts of the Hopper-specific SASS mnemonics (wgmma, TMA,
mbarrier) and of the main memory / FMA instructions.  usage: python tools/sass_summary.py > sass_summary.txt"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, 'c2-matching_b200', 'lib', 'libc2m_sm100.so')
out = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True, check=True).stdout
WANT = ['HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UBLKCP', 'SYNCS', 'HMMA', 'LDGSTS', 'ELECT',
        'UCGABAR', 'CCTL', 'SHFL', 'LDG', 'STG', 'LDS', 'STS', 'DFMA', 'FFMA', 'HFMA2']
cur, counts, total = None, collections.OrderedDict(), collections.Counter()
for ln in out.splitlines():
    m = re.search(r'Function : (\S+)', ln)
    if m:
        cur = subprocess.run(['c++filt', m.group(1)], capture_output=True, text=True).stdout.strip().split('(')[0]
        counts[cur] = collections.Counter()
        continue
    m = re.match(r'\s+/\*[0-9a-f]{4,6}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)', ln)
    if m and cur:
        op = m.group(1)
        total[cur] += 1
        for w in WANT:
            if op == w or op.startswith(w + '.') or (w in ('HGMMA', 'WARPGROUP', 'UTMALDG', 'SYNCS') and op.startswith(w)):
                counts[cur][w] += 1
print('# SASS instruction counts per kernel of c2-matching_b200/lib/libc2m_sm100.so (sm_90a; cuobjdump -sass)')
print('# HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / arrive, UTMALDG = cp.async.bulk.tensor (TMA load),')
print('# UBLKCP = cp.async.bulk, SYNCS = mbarrier ops, ELECT = elect.sync, HMMA = mma.sync\n')
for k, c in counts.items():
    if total[k] < 40 and not any(c[w] for w in ('HGMMA', 'UTMALDG')):
        continue
    print(f'{k}: {total[k]} instructions; ' + ', '.join(f'{w} {c[w]}' for w in WANT if c[w]))
