"""Per-CUDA-source-line stall samples (where warps WAIT) for one kernel of an .ncu-rep, plus the stall-reason totals:
   python scripts/ncu_stalls.py prof.ncu-rep <kernel index 1..> [topn]"""
import csv, subprocess, sys, collections
rep, kid = sys.argv[1], sys.argv[2]
topn = int(sys.argv[3]) if len(sys.argv) > 3 else 25
raw = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'sass,cuda', '--kernel-id', f':::{kid}'],
                     capture_output=True, text=True).stdout.splitlines()
inst = collections.Counter(); smp = collections.Counter(); reasons = collections.Counter(); cur = '?'; hdr = None
for l in raw:
    if l.startswith('"File Path"'):
        cur = l.split(',', 1)[1].strip('"').split('/')[-1]; hdr = None; continue
    if l.startswith('"Function Name"'): continue
    if l.startswith('"Line No"'):
        hdr = next(csv.reader([l])); ie = hdr.index('Instructions Executed'); isamp = hdr.index('# Samples'); isrc = hdr.index('Source')
        stall = [i for i, h in enumerate(hdr) if h.startswith('stall_') and 'Not Issued' not in h]; continue
    if hdr is None: continue
    r = next(csv.reader([l]))
    if len(r) < len(hdr) or not r[0].strip().isdigit(): continue
    try: n = int(r[ie]); s = int(r[isamp])
    except ValueError: continue
    key = (cur, int(r[0]), r[isrc].strip()[:100]); inst[key] += n; smp[key] += s
    for i in stall:
        try: reasons[hdr[i]] += int(r[i])
        except ValueError: pass
ti, ts = sum(inst.values()), sum(smp.values())
print(f'kernel {kid}: {ti:,} warp-instructions, {ts:,} samples')
print('stall reasons:', ', '.join(f'{k[6:]}={100*v/max(sum(reasons.values()),1):.1f}%' for k, v in reasons.most_common(10)))
for k, n in smp.most_common(topn):
    print(f'{100*n/ts:5.1f}% smp {100*inst[k]/ti:5.1f}% inst  {k[0][:14]:14s}:{k[1]:4d}  {k[2]}')
