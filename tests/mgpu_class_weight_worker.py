"""torchrun worker for tests/test_gpu_cbow_class_weight.py: an N-GPU full-batch run of the cbow_small golden windows
with class_weight="balanced" (resolved from the global training split, the same weights on every rank); rank 0 saves
the vectors."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(out):
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import g2vec_b200 as g2v
    from tests import helpers
    g = helpers.cbow_golden("cbow_small.npz")
    W, info = g2v.train_cbow(g["rowptr"], g["gene"], g["label"], g["V"], g["D"], g["lr"], max_epoch=10, seed=g["seed"],
                             log=None, early_stop=False, class_weight="balanced", return_info=True)
    w = torch.tensor(info["class_weight"], dtype=torch.float64, device="cuda")
    every = [torch.empty_like(w) for _ in range(dist.get_world_size())]
    dist.all_gather(every, w)
    assert all(torch.equal(e, w) for e in every)
    if dist.get_rank() == 0:
        np.save(out, W)
    dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
