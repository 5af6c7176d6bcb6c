# BASELINE config 5: sim-step sweep over the replica count (uniform-random actions), 1 GPU
OUT=${OUT:-results}; mkdir -p "$OUT"; export OUT      # output directory (git ignores results/)
for R in 256 1024 4096 8192 16384 32768 65536 131072; do
  python bench.py --mode sim --replicas $R --steps 60 --warmup 5 --burnin 240 --no-cpu-baseline 2>/dev/null | tail -1 > $OUT/sweep_$R.json
  python - <<PY
import json
d=json.load(open("$OUT/sweep_$R.json"))
print($R, round(d["value"]/1e6,1), "M steps/s", round(d["ms_per_step"],3), "ms", "roofline", round(d["roofline"]["frac"],4), "e2e", round(d["e2e"]["value"]/1e6,1))
PY
done
