OUT=${OUT:-results}; mkdir -p "$OUT"; export OUT      # output directory (git ignores results/)
ncu --metrics gpu__time_duration.sum --clock-control none -s ${LLS:-130} -c ${LLC:-745} --csv --log-file $OUT/ll.csv \
    python bench.py --replicas ${LLR:-2048} --burnin 120 --steps 121 --warmup 3 --no-cpu-baseline --profile-run > $OUT/ll.log 2>&1
python - <<'PY'
import csv, collections, os
rows=list(csv.reader(open(os.environ['OUT'] + '/ll.csv')))
i=[k for k,r in enumerate(rows) if r and r[0]=='ID'][0]
hdr=rows[i]; data=rows[i+1:]
kn=hdr.index('Kernel Name'); mv=hdr.index('Metric Value')
agg=collections.defaultdict(lambda:[0,0.0])
for r in data:
    if len(r)<=mv: continue
    n=r[kn][:100]; agg[n][0]+=1; agg[n][1]+=float(r[mv])
tot=sum(v[1] for v in agg.values())
for n,(c,t) in sorted(agg.items(), key=lambda x:-x[1][1])[:16]:
    print(f"{t/1e6:9.2f} ms {100*t/tot:5.1f}% x{c:5d}  {n}")
print('total ms', tot/1e6, len(data))
PY
