"""torchrun worker for tests/test_gpu_cbow_lr_plateau.py: an N-GPU full-batch run with the reduce-on-plateau learning
rate (lr_patience 1, factor 0.5) on the ex_* windows, once with the NVLink counter exchange (g2v_cbow_loop_counters_nvl)
and once with NCCL; rank 0 saves the vectors, the validation counts and every rank's rate record."""
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
    from tests import helpers, lr_plateau_oracle
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    W0, Wo0 = helpers.init_weights(7523, 128, 0)
    res, exchange = {}, []
    for name, env in (("nvl", {}), ("nccl", {"G2V_CBOW_NVL": "0"})):
        os.environ.update(env)
        W, info = g2v.train_cbow(rowptr, gene, label, 7523, 128, 0.005, max_epoch=20, seed=0, W_ih0=W0, W_ho0=Wo0,
                                 log=None, return_info=True, early_stop=False, lr_patience=1, lr_factor=0.5)
        for k in env:
            os.environ.pop(k)
        rates = torch.tensor(info["lr"], dtype=torch.float64, device="cuda")
        every = [torch.empty_like(rates) for _ in range(dist.get_world_size())]
        dist.all_gather(every, rates)
        res.update({name + "_W": W, name + "_lr": torch.stack(every).cpu().numpy(),
                    name + "_val": np.array(lr_plateau_oracle.val_counts(info), np.int64)})
        exchange.append(info["exchange"])
    if dist.get_rank() == 0:
        np.savez(out, exchange=np.array(exchange), **res)
    dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
