# round-end verification on one H100: GPU test suite, smoke, the headline bench and the supplementary bench lines
mkdir -p gpurun_out
set -x
timeout 900 python -m pytest tests -m gpu -q 2>&1 | tail -3
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
timeout 600 python bench.py 2>gpurun_out/final_err.log | tail -1 > gpurun_out/final_base.json
X="--no-cpu-baseline --hf-gpu-batches 0"
timeout 300 python bench.py --batch 512 $X 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_base_b512.json
timeout 300 python bench.py --lengths alpaca $X 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_base_alpaca.json
timeout 300 python bench.py --model flan-t5-small $X 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_small.json
timeout 400 python bench.py --model flan-t5-large $X --steps 2 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_large.json
timeout 300 python bench.py --dtype fp16 $X 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_fp16.json
timeout 600 python bench.py --impl reference --steps 1 --warmup 0 2>>gpurun_out/final_err.log | tail -1 > gpurun_out/final_reference_arm.json
set +x
for f in base base_b512 base_alpaca small large fp16; do python - <<PY
import json
try:
    d=json.load(open("gpurun_out/final_$f.json"))
    print("$f", round(d["ms_per_step"],1), "ms", round(d["value"]), "tok/s e2e", round(d["e2e"]["value"]), [round(x,1) for x in d["e2e"].get("ms_per_step_min_median_max",[])], "roofline", round(d["roofline"]["frac"],3), d["roofline"]["kernel"][:48], "decode", round(d["decode_loop"]["ms"],1), round(d["decode_loop"]["frac_of_hbm_peak"],3), "enc", round(d["encoder"]["ms"],1), round(d["encoder"]["frac_of_bf16_sustained"],3), d["clocks"]["reasons"], "parity", d.get("parity",{}).get("rows_equal_up_to_first_near_tie"), d.get("parity",{}).get("token_agreement"))
except Exception as e:
    print("$f FAILED", e)
PY
done
cat gpurun_out/final_reference_arm.json | cut -c1-600
