"""cuobjdump -sass of libc2m_sm100.so -> per-kernel counts of the Hopper-specific SASS mnemonics (wgmma, TMA,
mbarrier) and of the main memory / FMA instructions.  usage: python tools/sass_summary.py > sass_summary.txt

With --against OTHER.so it instead prints, for every kernel of either library, whether its SASS matches OTHER's:
instruction text only (addresses and the /* 0x... */ encodings are dropped), kernels paired by mangled name with the
anonymous-namespace hash (_GLOBAL__N__<hash>, which changes whenever a source file does) normalised away.  The exit
status is 1 when any kernel differs or exists in one library only."""
import argparse, collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'c2-matching_b200', 'lib', 'libc2m_sm100.so')
WANT = ['HGMMA', 'WARPGROUP', 'UTMALDG', 'UTMASTG', 'UBLKCP', 'SYNCS', 'HMMA', 'LDGSTS', 'ELECT',
        'UCGABAR', 'CCTL', 'SHFL', 'LDG', 'STG', 'LDS', 'STS', 'DFMA', 'FFMA', 'HFMA2']


def kernels(lib):
    """{normalised mangled name: (mangled name, [instruction text, ...])} of every function in the library's SASS"""
    out = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for ln in out.splitlines():
        m = re.search(r'Function : (\S+)', ln)
        if m:
            cur = funcs.setdefault(normalise(m.group(1)), (m.group(1), []))[1]
            continue
        m = re.match(r'\s+/\*[0-9a-f]{4,6}\*/\s+(.*?)\s*;?\s*/\* 0x[0-9a-f]+ \*/\s*$', ln)
        if m and cur is not None:
            cur.append(normalise(re.sub(r'\s+', ' ', m.group(1))))
    return funcs


def normalise(s):
    """drop the two hashes of an anonymous namespace's name, e.g. _GLOBAL__N__ffcf66d9_9_dcn_v2_cu_09059559"""
    return re.sub(r'_GLOBAL__N__[0-9a-f]{8}_(\d+_\w+?_cu)_[0-9a-f]{8}', r'_GLOBAL__N__\1', s)


def demangle(name):
    return subprocess.run(['c++filt', name], capture_output=True, text=True).stdout.strip()


def summary(lib):
    print(f'# SASS instruction counts per kernel of {os.path.relpath(lib, ROOT)} (sm_90a; cuobjdump -sass)')
    print('# HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / arrive, UTMALDG = cp.async.bulk.tensor (TMA load),')
    print('# UBLKCP = cp.async.bulk, SYNCS = mbarrier ops, ELECT = elect.sync, HMMA = mma.sync\n')
    for mangled, ins in kernels(lib).values():
        c = collections.Counter()
        for i in ins:
            op = re.match(r'(?:@!?U?P\d+\s+)?([A-Z0-9_]+)', i).group(1)
            for w in WANT:
                if op == w or op.startswith(w + '.') or (w in ('HGMMA', 'WARPGROUP', 'UTMALDG', 'SYNCS') and op.startswith(w)):
                    c[w] += 1
        if len(ins) < 40 and not any(c[w] for w in ('HGMMA', 'UTMALDG')):
            continue
        print(f'{demangle(mangled).split("(")[0]}: {len(ins)} instructions; ' + ', '.join(f'{w} {c[w]}' for w in WANT if c[w]))


def against(lib, other):
    a, b = kernels(lib), kernels(other)
    bad = 0
    for name in list(a) + [n for n in b if n not in a]:
        if name not in b or name not in a:
            verdict = 'only in ' + ('this library' if name in a else 'OTHER')
        elif a[name][1] == b[name][1]:
            verdict = f'identical ({len(a[name][1])} instructions)'
        else:
            verdict = f'DIFFERS ({len(b[name][1])} -> {len(a[name][1])} instructions)'
        bad += not verdict.startswith('identical')
        print(f'{demangle((a.get(name) or b[name])[0])}: {verdict}')
    print(f'# {len(set(a) | set(b)) - bad} identical, {bad} not')
    return 1 if bad else 0


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--lib', default=LIB, help='library to read (default: this tree\'s build)')
    ap.add_argument('--against', metavar='OTHER.so', help='compare every kernel\'s SASS with this library\'s')
    args = ap.parse_args()
    if args.against:
        sys.exit(against(args.lib, args.against))
    summary(args.lib)
