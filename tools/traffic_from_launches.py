"""ncu launch list of tools/one_step.py with
    --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum
-> (1) the per-kernel table of one steady-state step (stdout, markdown) and (2) profiles/dominant_kernel_traffic.json:
per kernel class the MEAN DRAM bytes per launch over the launches of that step — what bench.py reports as
`roofline.traffic` next to the per-launch `achieved` (the class's launches differ in shape, so both are class means).
usage: python tools/traffic_from_launches.py gpurun_out/launches.csv profiles/dominant_kernel_traffic.json"""
import collections, csv, json, sys

UNIT = {'ns': 1e-6, 'us': 1e-3, 'ms': 1.0, 'nsecond': 1e-6, 'usecond': 1e-3, 'msecond': 1.0, 's': 1e3, 'second': 1e3,
        'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9, 'Tbyte': 1e12}
with open(sys.argv[1]) as f:
    lines = [ln for ln in f if not ln.startswith('==')]
launches = collections.OrderedDict()          # ID -> {name, ms, rd, wr}
for r in csv.DictReader(lines):
    d = launches.setdefault(r['ID'], {'name': r['Kernel Name'].split('(')[0], 'ms': 0.0, 'rd': 0.0, 'wr': 0.0})
    v = float(r['Metric Value'].replace(',', '')) * UNIT[r['Metric Unit']]
    if r['Metric Name'] == 'gpu__time_duration.sum':
        d['ms'] = v
    elif r['Metric Name'] == 'dram__bytes_read.sum':
        d['rd'] = v
    elif r['Metric Name'] == 'dram__bytes_write.sum':
        d['wr'] = v
rows = list(launches.values())
corr = [i for i, d in enumerate(rows) if 'corr_umma_kernel' in d['name']]
step = rows[corr[-2]:corr[-1]]
acc = collections.OrderedDict()
for d in step:
    a = acc.setdefault(d['name'], [0, 0.0, 0.0, 0.0])
    a[0] += 1; a[1] += d['ms']; a[2] += d['rd']; a[3] += d['wr']
tot = sum(a[1] for a in acc.values())
print(f'# launches in step: {len(step)}   summed device time (serialised, cold cache): {tot:.2f} ms   DRAM read+write: '
      f'{sum(a[2] + a[3] for a in acc.values()) / 1e9:.2f} GB\n')
print('| kernel | launches | ms | share | DRAM read MB | DRAM write MB | MB per launch |\n|---|---:|---:|---:|---:|---:|---:|')
for k, a in sorted(acc.items(), key=lambda kv: -kv[1][1]):
    print(f'| `{k[:70]}` | {a[0]} | {a[1]:.3f} | {a[1] / tot * 100:.1f}% | {a[2] / 1e6:.0f} | {a[3] / 1e6:.0f} | {(a[2] + a[3]) / a[0] / 1e6:.1f} |')
if len(sys.argv) > 2:
    per = {}                                  # kernel -> [launches, bytes] over all its template instances
    for k, a in acc.items():
        short = k.split('<')[0].split('::')[-1]
        if short in ('conv3x3_wgmma_kernel', 'corr_umma_kernel', 'dcn_wgmma_kernel'):
            p = per.setdefault(short, [0, 0.0])
            p[0] += a[0]; p[1] += a[2] + a[3]
    out = {k: b / n for k, (n, b) in per.items()}
    out['note'] = ('mean dram__bytes_read.sum + dram__bytes_write.sum per launch over the launches of one steady-state bench step '
                   '(B=4 config 2), from the ncu launch list summarised in profiles/r02_launches_step.md')
    json.dump(out, open(sys.argv[2], 'w'), indent=1)
