"""Worker process of the two-GPU store audit (torchrun, one process per GPU): runs ShardedChecker on the CUDA shard
engine and dumps this rank's store for tests/test_zz_store_audit.py -- states, parent words, the new states of every
level on this rank, stats, coverage and violation record -- to <out_dir>/rank<r>.npz; rank 0 also writes the
job's result to <out_dir>/result.json."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "support"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from kafka_specification_b200.sharded import CudaShardEngine, ShardedChecker  # noqa: E402
from store_audit import copy_parents  # noqa: E402


class RecordingEngine(CudaShardEngine):
    """Keeps the number of new states each level end leaves on this rank (both level-end paths of the driver)."""
    level_counts: list

    def level_done(self):
        first, count = super().level_done()
        self.level_counts.append(count)
        return first, count

    def level_sync(self):
        board = super().level_sync()
        self.level_counts.append(board[self.rank][1])
        return board


def main():
    model, out_dir = sys.argv[1], sys.argv[2]
    cont = "cont" in sys.argv[3:]
    p2p = "nccl" not in sys.argv[3:]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    eng = RecordingEngine(model, rank, world, local, table_log2=22, max_states=2_000_000, p2p=p2p)
    eng.level_counts = []
    res = ShardedChecker(eng, cont=cont).run()
    ck = eng.ck
    st = ck.stats()
    n = st["distinct"]
    v = ck.violation()
    rec = ck.violation_record() if v else None
    cov = ck.coverage()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), states=ck.copy_states(0, n), parents=copy_parents(ck, 0, n),
             level_counts=np.asarray(eng.level_counts, dtype=np.int64),
             meta=json.dumps({"stats": st, "violation": v, "record": rec, "coverage": cov}))
    if rank == 0:
        with open(os.path.join(out_dir, "result.json"), "w") as f:
            json.dump({"levels": res.levels, "complete": res.complete, "violation": res.violation,
                       "distinct": res.distinct, "generated": res.generated, "p2p": eng.p2p}, f)
    dist.barrier()
    eng.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
