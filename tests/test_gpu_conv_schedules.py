"""Both consumer schedules of the tensor-core convolution, and every epilogue under the ping-pong one, are reached by the
launches of the benchmarked plans (read from the launcher's log, as test_tensor_core_variants_reached does)."""
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def test_conv_schedules_reached(lib):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, XUNET_CONV_LOG='1')
    r = subprocess.run([sys.executable, '-c', 'from tests.test_gpu_plan_launches import _launch_all_convs; _launch_all_convs()'],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    seen = set()
    for line in r.stderr.splitlines():
        if line.startswith('conv_tc mode='):
            kv = dict(re.findall(r'(\w+)=(\w+)', line))
            seen.add((kv['sched'], int(kv['BN']), int(kv['epi']), int(kv['tma_store'])))
    print('conv_tc (sched, BN, epi, tma_store) seen:', sorted(seen))
    # the schedule follows from the tile width alone
    assert all((s == 'pingpong') == (bn < 64) for s, bn, _, _ in seen), sorted(seen)
    reached = {
        'cooperative': any(s == 'cooperative' for s, _, _, _ in seen),
        'pingpong TMA-store epilogue': any(s == 'pingpong' and t == 1 for s, _, _, t in seen),
        **{f'pingpong EPI {e}': any(s == 'pingpong' and ep == e for s, _, ep, _ in seen) for e in range(4)},
    }
    for k, v in reached.items():
        print(f'  {k}: {"reached" if v else "NOT reached"}')
    assert all(reached.values()), [k for k, v in reached.items() if not v]
