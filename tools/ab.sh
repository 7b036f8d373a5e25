# same-box A/B of two builds of libb200spark.so (old copy at dash-infer_b200/lib/libb200spark_old.so)
L=dash-infer_b200/lib
cp $L/libb200spark.so /tmp/new.so
run() { timeout 600 python tools/gemm_balance.py 2>&1 | grep -v "^#"; timeout 300 python bench.py --gpus 1 --no-cpu --steps 100 --warmup 10 2>&1 | tail -1 | python -c "import sys,json; d=json.loads(sys.stdin.read()); print(d['ms_per_step'], {k.split('[')[1][:6]:v['us'] for k,v in d['kernels'].items()})"; }
echo "== OLD"; cp $L/libb200spark_old.so $L/libb200spark.so; run
echo "== NEW"; cp /tmp/new.so $L/libb200spark.so; run
