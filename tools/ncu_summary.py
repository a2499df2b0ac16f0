"""Summarises an .ncu-rep (ncu --set full) into a markdown table.
  python tools/ncu_summary.py igemm_full.ncu-rep igemm_full.md "title"
"""
import csv
import io
import subprocess
import sys

WANT = [
    ('gpu__time_duration.sum', 'us', 1e-3),
    ('dram__bytes_read.sum', 'MB rd', None),
    ('dram__bytes_write.sum', 'MB wr', None),
    ('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 'dram %', 1),
    ('lts__t_bytes.sum', 'L2 MB', None),
    ('lts__throughput.avg.pct_of_peak_sustained_elapsed', 'L2 %', 1),
    ('sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active', 'tensor %', 1),
    ('sm__inst_executed_pipe_tensor_op_hmma.avg.pct_of_peak_sustained_active', 'tensor inst %', 1),
    ('sm__throughput.avg.pct_of_peak_sustained_elapsed', 'SM %', 1),
    ('launch__registers_per_thread', 'regs', 1),
    ('launch__grid_size', 'grid', 1),
]


def to_bytes(val, unit):
  v = float(val.replace(',', ''))
  u = unit.lower()
  mult = {'byte': 1, 'kbyte': 1e3, 'mbyte': 1e6, 'gbyte': 1e9, 'tbyte': 1e12}.get(u, 1)
  return v * mult


def main():
  rep, out, title = sys.argv[1], sys.argv[2], sys.argv[3]
  raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], stdout=subprocess.PIPE, text=True).stdout
  rows = list(csv.reader(io.StringIO(raw)))
  hdr, units = rows[0], rows[1]
  col = {h: i for i, h in enumerate(hdr)}
  names = [n for n, _, _ in WANT if n in col]
  missing = [n for n, _, _ in WANT if n not in col]
  tensor_cols = [h for h in hdr if 'tensor' in h and 'pct' in h]
  agg = {}
  lines = []
  for r in rows[2:]:
    if len(r) < len(hdr):
      continue
    kname = r[col['Kernel Name']].split('(')[0]
    vals = {}
    for n in names:
      v, u = r[col[n]], units[col[n]]
      if not v:
        continue
      if 'bytes' in n:
        vals[n] = to_bytes(v, u) / 1e6
      elif n == 'gpu__time_duration.sum':
        f = float(v.replace(',', ''))
        vals[n] = f / 1e3 if u in ('ns', 'nsecond') else (f if u in ('us', 'usecond') else f * 1e3)
      else:
        vals[n] = float(v.replace(',', ''))
    extra = {h: r[col[h]] for h in tensor_cols[:3]}
    lines.append((kname, vals, extra))
    a = agg.setdefault(kname, {'n': 0})
    a['n'] += 1
    for k, v in vals.items():
      a[k] = a.get(k, 0.0) + v
  with open(out, 'w') as f:
    f.write('# %s\n\nSource: `%s` (ncu --set full --clock-control none; per-launch values are cold-cache, serialised).\n\n' % (title, rep))
    if missing:
      f.write('Metrics not present in this capture: %s\n\n' % ', '.join(missing))
    f.write('## Per kernel (sums over launches; %% columns are launch-time-weighted means)\n\n')
    f.write('| kernel | launches | time ms | DRAM rd MB | DRAM wr MB | DRAM % | L2 MB | L2 % | tensor % | SM % |\n|---|---|---|---|---|---|---|---|---|---|\n')
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1].get('gpu__time_duration.sum', 0)):
      t = a.get('gpu__time_duration.sum', 0.0)
      def wmean(metric):
        num = sum(v.get(metric, 0.0) * v.get('gpu__time_duration.sum', 0.0) for kk, v, _ in lines if kk == k)
        return num / t if t else 0.0
      f.write('| `%s` | %d | %.3f | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f |\n' % (
          k[:70], a['n'], t / 1e3, a.get('dram__bytes_read.sum', 0), a.get('dram__bytes_write.sum', 0),
          wmean('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed'), a.get('lts__t_bytes.sum', 0),
          wmean('lts__throughput.avg.pct_of_peak_sustained_elapsed'),
          wmean('sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active') or
          wmean('sm__inst_executed_pipe_tensor_op_hmma.avg.pct_of_peak_sustained_active'),
          wmean('sm__throughput.avg.pct_of_peak_sustained_elapsed')))
    f.write('\n## Slowest 25 launches\n\n| kernel | us | DRAM rd MB | DRAM wr MB | DRAM % | L2 % | tensor % | grid | regs |\n|---|---|---|---|---|---|---|---|---|\n')
    for k, v, _ in sorted(lines, key=lambda x: -x[1].get('gpu__time_duration.sum', 0))[:25]:
      f.write('| `%s` | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f | %d | %d |\n' % (
          k[:60], v.get('gpu__time_duration.sum', 0), v.get('dram__bytes_read.sum', 0), v.get('dram__bytes_write.sum', 0),
          v.get('gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed', 0),
          v.get('lts__throughput.avg.pct_of_peak_sustained_elapsed', 0),
          v.get('sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active',
                v.get('sm__inst_executed_pipe_tensor_op_hmma.avg.pct_of_peak_sustained_active', 0)),
          int(v.get('launch__grid_size', 0)), int(v.get('launch__registers_per_thread', 0))))
    tot_rd = sum(a.get('dram__bytes_read.sum', 0) for a in agg.values())
    tot_wr = sum(a.get('dram__bytes_write.sum', 0) for a in agg.values())
    f.write('\nTotal DRAM traffic of the captured launches: %.1f MB read + %.1f MB written = %.1f MB\n' % (tot_rd, tot_wr, tot_rd + tot_wr))
    f.write('\nTensor-related metric columns present: %s\n' % ', '.join(tensor_cols[:12]))
  print('wrote', out)


if __name__ == '__main__':
  main()
