"""Multi-GPU check of the poisson Laplace-Vecchia path, run under torchrun (one process per GPU):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/mgpu_poisson_check.py
Every rank holds the whole latent factor and runs its share of the SLQ probe columns; the mean residual norm of each SLQ iteration
and the quadrature sum are all-reduced (gpbdev_vecchia_laplace_set_collective). The likelihood must match the reference's goldens
(tests/golden/laplace_poisson_golden.json) at the single-GPU bar. The gradient, and with it a fit, refuses probe columns sharded
over ranks (as for bernoulli_logit): the check asserts that refusal."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import poisson_data  # noqa: E402
from gpboost_b200 import GPModel, load_lib  # noqa: E402
from gpboost_b200.basic import GPBoostError  # noqa: E402
from gpboost_b200.parallel import init_nccl  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    lib = load_lib()
    init_nccl(lib, dist, local)
    log = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    gold = json.load(open(os.path.join(HERE, "golden", "laplace_poisson_golden.json")))["cases"]
    for c in gold:
        X, y, off = poisson_data.case_data(c)
        gm = GPModel(likelihood="poisson", gp_coords=X, cov_function=c["cov_function"], cov_fct_shape=c["shape"], gp_approx="vecchia",
                     num_neighbors=c["m"], vecchia_ordering=c["ordering"], seed=c["seed"], matrix_inversion_method="iterative")
        gm.set_optim_params(dict(num_rand_vec_trace=c["t"]))
        v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
        assert abs(v - c["negll"]) <= 1e-6 * abs(c["negll"]), (c["name"], v, c["negll"])
        assert int(gm.laplace_info()[1]) == c["newton_it"], (c["name"], gm.laplace_info(), c["newton_it"])
        log("poisson nll sharded ok: %s %.10g" % (c["name"], v))
    try:
        gm.fit(y, offset=off)
        raise AssertionError("a fit with sharded probe columns should have been refused")
    except GPBoostError as e:
        assert "sharded over ranks" in str(e), str(e)
    log("poisson fit with sharded probe columns refused as expected")
    dist.barrier()
    log("MGPU POISSON OK world=%d" % world)
    lib.GPB200_NcclFinalize()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
