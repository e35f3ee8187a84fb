"""bench.py's driver contract on a machine without a GPU: the reference arm (`--impl reference`: the reference's own code from
the checkout named by DBOA_REFERENCE_ROOT through oracle/ref_harness.py, else the CPU port of the path) prints ONE JSON line with the keys the driver reads, and our own arm fails loudly instead of falling back."""
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(*args, env=None):
    return subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), *args], capture_output=True, text=True, timeout=600, cwd=REPO,
                          env=dict(os.environ, **(env or {})))


def test_reference_arm_prints_the_contract_line():
    r = run('--impl', 'reference', '--steps', '1', '--warmup', '0')
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('{')]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for key in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling', 'vs_baseline', 'dtype',
                'data', 'config', 'e2e', 'cpu_baseline', 'impl'):
        assert key in d, key
    assert d['impl'] == 'reference' and d['unit'] == 'frames/s' and d['higher_is_better'] is True and d['vs_baseline'] is None
    assert d['value'] > 0 and d['steps'] == 1 and d['gpu_launches'] == 0
    assert d['cpu_baseline']['kind'] in ('reference', 'port') and d['cpu_baseline']['cores'] >= 1
    assert d['e2e']['value'] == d['value'] and d['e2e']['h2d_bytes_per_step'] == 0 and d['e2e']['d2h_bytes_per_step'] == 0
    assert 'workload' in d['config'] and 'model' not in d['config']


def test_reference_arm_falls_back_to_the_port_without_a_reference_tree():
    r = run('--impl', 'reference', '--steps', '1', '--warmup', '0', env={'DBOA_REFERENCE_ROOT': 'none'})
    assert r.returncode == 0, r.stderr[-2000:]
    d = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith('{')][0])
    assert d['cpu_baseline']['kind'] == 'port' and d['value'] > 0


def test_own_arm_needs_a_gpu_and_says_so():
    import torch
    if torch.cuda.is_available():
        return
    r = run('--steps', '1', '--warmup', '3')
    assert r.returncode != 0                                   # no silent CPU fallback
    assert 'cuda' in (r.stderr + r.stdout).lower()
