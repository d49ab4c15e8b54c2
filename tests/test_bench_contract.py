"""CPU: the committed bench lines carry every key of the bench contract, and bench.py parses without a GPU."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

REQUIRED = ['metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
            'vs_baseline', 'dtype', 'data', 'config', 'e2e', 'gpu_launches', 'clocks', 'roofline']


def _load(name):
    return json.load(open(os.path.join(ROOT, 'profiles', name)))


def test_own_arm_line_has_the_contract_keys():
    d = _load('bench_h100_cfg3.json')
    for k in REQUIRED + ['cpu_baseline']:
        assert k in d, k
    base = json.load(open(os.path.join(ROOT, 'BASELINE.json')))
    assert d['metric'] in base['metric'] and d['unit'] == 'tuples/s' and d['higher_is_better'] is True
    assert d['scaling'] == 'weak' and d['vs_baseline'] is None and d['data'] == 'synthetic'
    assert 'workload' in d['config'] and 'model' not in d['config']
    assert d['warmup'] >= 3 and d['gpu_launches'] > 0
    e = d['e2e']
    assert e['h2d_bytes_per_step'] > 0 and e['d2h_bytes_per_step'] > 0 and e['value'] != d['value']
    r = d['roofline']
    for k in ('bound', 'achieved', 'peak', 'unit', 'frac', 'traffic'):
        assert k in r, k
    assert r['bound'] in ('hbm', 'tensor') and abs(r['frac'] - r['achieved'] / r['peak']) < 1e-9
    assert d['value'] > 100 and d['run']['attention_split'] == 'fp16 hi/lo'     # 1 x H100 SXM at a 400 W power limit
    p = d['pose_auc_parity']
    assert p['max_abs_diff_pt'] <= 0.5 and p['n_errors'] == 320
    c = d['cpu_baseline']
    assert c['kind'] in ('reference', 'port') and c['cores'] >= 1 and c['sample']
    assert not set(d['clocks']['reasons']) & {'hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown'}


def test_bench_cli_parses_without_gpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--help'], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and '--impl' in r.stdout and '--gpus' in r.stdout
