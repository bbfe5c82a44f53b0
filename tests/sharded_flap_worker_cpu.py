"""gloo worker for tests/test_flap_cpu.py: a sharded pool (host emulation, 2 ranks) refuses flap schedules with
GSIM_ERR_STATE on every rank and runs on unchanged."""
import os
import sys

import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from consul_b200 import _lib  # noqa: E402
from consul_b200.pool import GsimError, lan_config  # noqa: E402
from consul_b200.sharded import ShardedPool  # noqa: E402

dist.init_process_group("gloo")
rank = dist.get_rank()
L = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
N = 2 * 4096
p = ShardedPool(lan_config(L, capacity=N, n_initial=N, seed=0x5A4E), L)
codes = []
for op in (lambda: p.impair_flap([1, 2], 10, 500000), lambda: p.impair_flap_fraction(10000, 1, 10, 500000),
           lambda: p.impair_flap_get(1), lambda: p.flap_stats()):
    try:
        op()
        codes.append(0)
    except GsimError as e:
        codes.append(e.code)
p.step(20)
ok = codes == [-6, -6, -6, -6] and p.stats()["suspects"] == 0
p.close()
if ok and rank == 0:
    print("FLAP REFUSED", flush=True)
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
