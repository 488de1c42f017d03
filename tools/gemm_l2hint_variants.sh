for h in 0 1 2 3; do
  FSB_GEMM_L2HINT=$h timeout 100 ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none -k regex:gemm_bf16 -s 2 -c 1 --csv python tools/prof_gemm.py NT 8192 15360 5120 2>/dev/null | grep -E "dram__bytes|time_duration" | awk -F'","' -v h=$h '{print "hint="h, $(NF-2), $NF}'
done
for h in 0 1 2 3; do echo L2HINT=$h; FSB_GEMM_L2HINT=$h timeout 100 python tools/bench_gemm.py 2>&1 | grep -E "llama (qkv|w13 fwd|w2 fwd|w13 wgrad)" | cut -c1-100; done
