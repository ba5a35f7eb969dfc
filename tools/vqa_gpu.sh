timeout 900 python -m pytest tests/test_gpu_parity.py -x -q -m gpu -k "vqa or real_size or golden" 2>&1 | tail -5
timeout 300 python bench.py --config vqa514 --steps 20 --warmup 5 --no-cpu-baseline --no-e2e 2>/dev/null | python -c "
import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); print('vqa514', d['value'], d['kernel_us'])"
