"""gloo worker for tests/test_domain_cpu.py: a sharded pool (host emulation, 2 ranks) refuses every fault-domain
call with GSIM_ERR_STATE on every rank and runs on unchanged."""
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
for op in (lambda: p.domain_set([1, 2], 3), lambda: p.domain_set_range(0, 64, 32, 1), lambda: p.domains(0, 4),
           lambda: p.domain_flap([1], 10, 500000), lambda: p.domain_flap_get(1), lambda: p.domain_impair([1], 10, 10),
           lambda: p.domain_crash([1]), lambda: p.domain_pause([1], 5), lambda: p.domain_stats(1, 2)):
    try:
        op()
        codes.append(0)
    except GsimError as e:
        codes.append(e.code)
p.step(20)
ok = codes == [-6] * 9 and p.stats()["suspects"] == 0
p.close()
if ok and rank == 0:
    print("DOMAINS REFUSED", flush=True)
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
