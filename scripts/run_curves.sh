set -x
OUT=${OUT:-results}; mkdir -p "$OUT"; export OUT      # output directory (git ignores results/)
python scripts/train_curve.py --replicas 512 --episodes 4 --greedy --tag greedy_grid > $OUT/tc_greedy.log 2>&1
python scripts/profile_policy_phases.py > $OUT/r02_policy_phases.log 2>&1
python scripts/train_curve.py --replicas 512 --episodes 600 --agent ma2c --tag ma2c_grid_bf16 > $OUT/tc_bf16.log 2>&1
python scripts/train_curve.py --replicas 512 --episodes 600 --agent ma2c --fp32 --tag ma2c_grid_fp32 > $OUT/tc_fp32.log 2>&1
python scripts/train_curve.py --replicas 512 --episodes 600 --agent ma2c --reward-norm 250 --tag ma2c_grid_bf16_rn250 > $OUT/tc_rn250.log 2>&1
python scripts/train_curve.py --replicas 512 --episodes 600 --agent ma2c --fp32 --reward-norm 250 --tag ma2c_grid_fp32_rn250 > $OUT/tc_rn250_fp32.log 2>&1
timeout 400 python scripts/train_curve.py --replicas 1 --episodes 300 --agent ma2c --tag ma2c_grid_R1 > $OUT/tc_r1.log 2>&1
tail -2 $OUT/tc_*.log
