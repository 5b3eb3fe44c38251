"""torchrun worker for tests/test_gpu_cbow_val_loss.py: an N-GPU full-batch run monitoring the validation loss (patience
3, lr_patience 1) on the ex_* windows, once with the NVLink score exchange (g2v_cbow_loop_score_nvl) and once with NCCL;
rank 0 saves the vectors, every rank's per-step loss and the stop and best steps."""
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
    (rowptr, gene, label), _ = helpers.ex_windows(reps=2)
    W0, Wo0 = helpers.init_weights(7523, 128, 0)
    res, exchange = {}, []
    for name, env in (("nvl", {}), ("nccl", {"G2V_CBOW_NVL": "0"})):
        os.environ.update(env)
        W, info = g2v.train_cbow(rowptr, gene, label, 7523, 128, 0.005, max_epoch=30, seed=0, W_ih0=W0, W_ho0=Wo0,
                                 log=None, return_info=True, patience=3, lr_patience=1, lr_factor=0.5,
                                 monitor="val_loss")
        for k in env:
            os.environ.pop(k)
        loss = torch.tensor(info["val_loss"], dtype=torch.float64, device="cuda")
        every = [torch.empty_like(loss) for _ in range(dist.get_world_size())]
        dist.all_gather(every, loss)
        res.update({name + "_W": W, name + "_loss": torch.stack(every).cpu().numpy(),
                    name + "_steps": np.array([-1 if info["stop_step"] is None else info["stop_step"],
                                               info["best_step"]], np.int64)})
        exchange.append(info["exchange"])
    if dist.get_rank() == 0:
        np.savez(out, exchange=np.array(exchange), **res)
    dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
