"""Multi-GPU parity check, run under torchrun (one process per GPU):
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/mgpu_check.py
Row-sharded Vecchia likelihood / fit, data-parallel boosting (histogram all-reduce), GPBoost iteration and the Laplace path with
sharded SLQ probe columns — every result against the golden vectors the single-GPU tests use. The collective is the C++ runtime's
own NCCL communicator (GPB200_NcclInit); torch.distributed only broadcasts the NCCL id."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import datagen  # noqa: E402
import treedata  # noqa: E402
from gpboost_b200 import GPModel, load_lib  # noqa: E402
from gpboost_b200.booster import Booster, Dataset, parse_model_string  # noqa: E402
from gpboost_b200.parallel import init_nccl  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    lib = load_lib()
    init_nccl(lib, dist, local)
    log = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)

    # ---- 1. Gaussian Vecchia: likelihood + fit, rows of the ordered observations sharded
    gold = json.load(open(os.path.join(HERE, "golden", "vecchia_golden.json")))
    from conftest import case_data
    nchk = 0

    def model_of(s):
        return GPModel(gp_coords=case_data(s)[0], cov_function=s["cov_function"], cov_fct_shape=s["cov_fct_shape"], gp_approx="vecchia",
                       num_neighbors=s["num_neighbors"], vecchia_ordering=s["vecchia_ordering"], seed=s.get("seed_model", s["seed"]))

    for s in gold["nll"]:
        coords, y = case_data(s)
        if coords.shape[0] < 200:
            continue
        v = model_of(s).neg_log_likelihood(np.array(s["cov_pars"]), y)
        assert abs(v - s["negll"]) <= 1e-9 * abs(s["negll"]), (s, v)
        nchk += 1
    log("vecchia nll sharded: %d cases ok" % nchk)
    s = [r for r in gold["fit"] if case_data(r)[0].shape[0] >= 1000][0]
    coords, y = case_data(s)
    m = model_of(s)
    m.fit(y)
    assert abs(m.get_current_neg_log_likelihood() - s["negll"]) <= 2e-6 * abs(s["negll"])
    g = m.response_gradient(y)
    m1 = np.array(g)  # Psi^-1 y must be identical on all ranks (n-vector all-reduced on the device)
    t = torch.from_numpy(m1.copy()).cuda(); dist.all_reduce(t, op=dist.ReduceOp.MAX)
    assert np.array_equal(t.cpu().numpy(), m1)
    log("vecchia fit sharded ok: negll %.10g" % m.get_current_neg_log_likelihood())

    # ---- 2. data-parallel boosting: histograms all-reduced per split, trees must equal the reference's
    tg = json.load(open(os.path.join(HERE, "golden", "tree_golden.json")))
    for rec in tg["cases"]:
        spec = rec["spec"]
        X, y, coords = treedata.make_case(spec)
        params = treedata.booster_params(spec, reference=False)
        gp = None
        if spec.get("gp"):
            gp = GPModel(gp_coords=coords, cov_function="matern", cov_fct_shape=1.5, gp_approx="vecchia", num_neighbors=spec["num_neighbors"],
                         vecchia_ordering="random", seed=1)
            if spec.get("init_cov_pars"):
                gp.set_optim_params({"init_cov_pars": np.array(spec["init_cov_pars"])})
        if spec.get("newton"):  # Newton leaf updates need the whole factor on one device: refused for row shards, through the error channel
            from gpboost_b200.basic import GPBoostError
            try:
                Booster(params, Dataset(X, y, params=params), gp_model=gp).update()
                raise AssertionError("leaves_newton_update with row shards should have been refused")
            except GPBoostError as e:
                assert "row-sharded" in str(e), str(e)
            continue
        b = Booster(params, Dataset(X, y, params=params), gp_model=gp)
        for _ in range(spec["num_iter"]):
            b.update()
        trees = parse_model_string(b.model_to_string())
        score = b.inner_predict_train()
        if spec.get("gp") and spec.get("train_cov") is not False:
            g0 = rec["trees"][0]
            assert np.array_equal(trees[0]["split_feature"], np.array(g0["split_feature"]))
            assert np.array_equal(trees[0]["threshold"], np.array(g0["threshold"]))
            cp = gp.get_cov_pars()
            assert np.all(np.abs(cp - np.array(rec["cov_pars"])) <= 5e-3 * np.abs(rec["cov_pars"])), (cp, rec["cov_pars"])
            assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 2e-3 * np.abs(rec["score_head"]).max()
        else:
            assert len(trees) == len(rec["trees"]), spec["name"]
            for tr, g in zip(trees, rec["trees"]):
                assert tr["num_leaves"] == g["num_leaves"], spec["name"]
                assert np.array_equal(tr["split_feature"], np.array(g["split_feature"])), spec["name"]
                assert np.array_equal(tr["threshold"], np.array(g["threshold"])), spec["name"]
                assert np.array_equal(tr["leaf_count"], np.array(g["leaf_count"])), spec["name"]
                assert np.max(np.abs(tr["leaf_value"] - np.array(g["leaf_value"]))) <= 1e-8 * np.max(np.abs(g["leaf_value"]))
            assert np.abs(score[:64] - np.array(rec["score_head"])).max() <= 1e-8 * np.abs(rec["score_head"]).max()
            assert abs(score.sum() - rec["score_sum"]) <= 1e-8 * max(abs(rec["score_sum"]), np.abs(score).sum() * 1e-3)
        log("boosting sharded ok:", spec["name"])

    # ---- 3. Laplace-Vecchia with the SLQ probe columns sharded over the ranks
    lg = json.load(open(os.path.join(HERE, "golden", "laplace_golden.json")))["cases"]
    for c in lg[1:4]:
        X, y, off = datagen.binary_synth(c["n"], c["dseed"], c["offset"])
        gm = GPModel(likelihood="bernoulli_logit", gp_coords=X, cov_function=c["cov_function"], cov_fct_shape=c["shape"], gp_approx="vecchia",
                     num_neighbors=c["m"], vecchia_ordering=c["ordering"], seed=c["seed"], matrix_inversion_method="iterative")
        v = gm.neg_log_likelihood(np.array(c["cov_pars"]), y, fixed_effects=off)
        assert abs(v - c["negll_iterative"]) <= 1e-6 * abs(c["negll_iterative"]), (v, c["negll_iterative"])
    log("laplace sharded ok")
    dist.barrier()
    log("MGPU OK world=%d" % world)
    lib.GPB200_NcclFinalize()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
