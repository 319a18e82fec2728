"""Per-CUDA-source-line share of executed instructions and stall samples for one kernel of an .ncu-rep:
   python scripts/ncu_lines.py prof.ncu-rep <kernel index 1..> [topn]"""
import csv, subprocess, sys, collections
rep, kid = sys.argv[1], sys.argv[2]
topn = int(sys.argv[3]) if len(sys.argv) > 3 else 40
raw = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'sass,cuda', '--kernel-id', f':::{kid}'],
                     capture_output=True, text=True).stdout.splitlines()
inst = collections.Counter(); smp = collections.Counter(); cur = '?'; hdr = None
for l in raw:
    if l.startswith('"File Path"'):
        cur = l.split(',', 1)[1].strip('"').split('/')[-1]; hdr = None; continue
    if l.startswith('"Function Name"'): continue
    if l.startswith('"Line No"'):
        hdr = next(csv.reader([l])); ie = hdr.index('Instructions Executed'); isamp = hdr.index('# Samples'); isrc = hdr.index('Source'); continue
    if hdr is None: continue
    r = next(csv.reader([l]))
    if len(r) < len(hdr) or not r[0].strip().isdigit(): continue      # keep only CUDA-source rows (they aggregate their SASS)
    try: n = int(r[ie]); s = int(r[isamp])
    except ValueError: continue
    key = (cur, int(r[0]), r[isrc].strip()[:100]); inst[key] += n; smp[key] += s
ti, ts = sum(inst.values()), sum(smp.values())
print(f'kernel {kid}: {ti:,} warp-instructions attributed, {ts:,} samples')
for k, n in inst.most_common(topn):
    print(f'{100*n/ti:5.1f}% inst {100*smp[k]/max(ts,1):5.1f}% smp  {k[0][:14]:14s}:{k[1]:4d}  {k[2]}')
