"""K5 at scale on one GPU: arrival-order load (stable group-by) + fold, stage times; then 100 k-record micro-batches through the
sort-based incremental path (the group-by's compact mode). Each line ends with a digest of the state table, so two builds can
be compared output for output.

    python scripts/group_prof.py [n_agg] [events per aggregate] [micro-batch steps]
"""
import hashlib, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from surge_b200 import ReplayEngine, programs as P
n_agg = int(sys.argv[1]) if len(sys.argv) > 1 else 1 << 20
epa = int(sys.argv[2]) if len(sys.argv) > 2 else 32
inc_steps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
dev = "cuda:0"
n = n_agg * epa
gen = torch.Generator(device=dev); gen.manual_seed(1)
r = torch.zeros((n, 16), dtype=torch.int32, device=dev)
agg = torch.arange(n_agg, device=dev, dtype=torch.int64).repeat(epa)   # event e of every aggregate before event e+1
u = torch.rand(n, generator=gen, device=dev)
r[:, 0] = torch.where(u < 0.45, 0, torch.where(u < 0.9, 1, 2)).to(torch.int32)
r[:, 1] = torch.arange(epa, device=dev, dtype=torch.int32).repeat_interleave(n_agg) + 1
r[:, 2] = agg.to(torch.int32)
r[:, 4] = torch.randint(0, 1 << 31, (n,), generator=gen, device=dev, dtype=torch.int64).to(torch.int32)
del agg, u


def digest(e):
    return hashlib.sha256(np.ascontiguousarray(e.export_states()).tobytes()).hexdigest()[:16]


e = ReplayEngine(0); e.register_program(P.counter_program())
for it in range(3):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    e.load_unsorted(r.view(torch.uint8), n_agg)
    torch.cuda.synchronize(); t1 = time.perf_counter()
    e.set_initial_states(None); e.fold()
    st = e.stats()
    print(f"n={n} records ({n*64/2**30:.2f} GiB) n_agg={n_agg}: group {st.ms_group:.3f} ms ({n*64*2/st.ms_group/1e6:.0f} GB/s of 2x record bytes) "
          f"fold {st.ms_fold:.3f} ms wall_load {1e3*(t1-t0):.2f} ms events={st.n_events} states={digest(e)}", flush=True)
# micro-batches of 100 k records drawn from the whole log, folded through the group-by (incremental = 1 bypasses the sort-free kernel)
e.set_option("incremental", 1)
nb = min(100_000, n)
groups = []
for it in range(inc_steps + 2):
    batch = r[torch.randint(0, n, (nb,), generator=gen, device=dev)].contiguous()
    e.fold_incremental(batch.view(torch.uint8))
    if it >= 2:   # the first two grow the scratch
        groups.append(e.stats().ms_group)
print(f"micro-batch n={nb} records n_agg={n_agg} x {len(groups)}: group median {np.median(groups):.4f} ms "
      f"min {min(groups):.4f} max {max(groups):.4f} states={digest(e)}", flush=True)
