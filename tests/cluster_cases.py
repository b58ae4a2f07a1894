"""Cases of the independent-realizations goldens (tests/golden/make_cluster_golden.py): Gaussian Vecchia GPs with `cluster_ids`, run
through the shared frontend on this build's library or, with `lib`, on the unmodified reference library.

Every model case has 3-5 clusters with unsorted labels that interleave in the data, of unequal sizes: one cluster with fewer than
num_neighbors + 1 points and one of a single point. It records the likelihood at fixed parameters, a fit (parameters, likelihood,
iterations) and the prediction (means and response variances) at points of every cluster and of a label without training data."""
import numpy as np

from gpboost_b200 import GPModel
from gpboost_b200.booster import Booster, Dataset

NEW_LABEL = 99  # a cluster without training data: predicted from the prior

# (name, labels with their sizes, num_neighbors, covariance, shape, ordering, seed)
CASES = [
    dict(name="exp_m10_none", labels=[7, 2, 5, 9, 4], sizes=[700, 400, 250, 8, 1], m=10, cov="matern", shape=0.5, ordering="none",
         seed=1),
    dict(name="m15_m30_random", labels=[7, 2, 5, 3], sizes=[1200, 500, 20, 1], m=30, cov="matern", shape=1.5, ordering="random", seed=2),
    # prediction with 60 neighbours, the device's limit (the default would be 2 m = 90)
    dict(name="m25_m45_random", labels=[3, 8, 1], sizes=[600, 400, 30], m=45, cov="matern", shape=2.5, ordering="random", seed=3, mp=60),
    dict(name="gauss_m30_none", labels=[5, 1, 6, 2], sizes=[500, 350, 12, 1], m=30, cov="gaussian", shape=0., ordering="none", seed=4),
    dict(name="m15_m20_random_one_big", labels=[4, 11, 6], sizes=[900, 150, 1], m=20, cov="matern", shape=1.5, ordering="random", seed=5),
]
COV_PARS = [0.2, 1.0, 0.1]  # error variance, marginal variance, range
NUM_PRED = 60

# GPBoost: trees at fixed covariance parameters (every tree) and with trained parameters (the first tree)
BOOST_CASE = dict(name="boost_exp_m10", labels=[6, 1, 3, 8], sizes=[500, 300, 7, 1], m=10, cov="matern", shape=0.5, ordering="random",
                  seed=6, F=4, num_leaves=8, num_it=5, nv=150)
# the same boosting at fixed covariance parameters with Newton leaf updates, which read the resident factor. (The line search of the step
# length is refused with cluster_ids: the reference library fails an index assertion in it for such a model.)
BOOST_VARIANTS = {"boost_newton": dict(leaves_newton_update=True)}


def labels_of(c, rng):
    """cluster label of every point: the case's labels with their sizes, in a random interleaving"""
    lab = np.concatenate([np.full(s, l, dtype=np.int32) for l, s in zip(c["labels"], c["sizes"])])
    return lab[rng.permutation(len(lab))]


def case_data(c):
    rng = np.random.default_rng(c["seed"])
    lab = labels_of(c, rng)
    n = len(lab)
    coords = rng.uniform(0., 1., size=(n, 2))
    shift = {l: rng.normal(0., 1.) for l in c["labels"]}
    y = np.array([np.sin(5. * coords[i, 0]) * np.cos(4. * coords[i, 1]) + 0.3 * shift[lab[i]] for i in range(n)])
    y = y + 0.3 * rng.standard_normal(n)
    # prediction points: in every training cluster and in a new one, interleaved
    lab_p = np.array([c["labels"][k % len(c["labels"])] if k % 7 else NEW_LABEL for k in range(NUM_PRED)], dtype=np.int32)
    lab_p = lab_p[rng.permutation(NUM_PRED)]
    coords_p = rng.uniform(0., 1., size=(NUM_PRED, 2))
    return coords, y, lab, coords_p, lab_p


def model_of(c, coords, lab, lib=None, cluster_ids=True):
    kw = {} if lib is None else dict(_lib=lib)
    return GPModel(gp_coords=coords, cov_function=c["cov"], cov_fct_shape=c["shape"], gp_approx="vecchia", num_neighbors=c["m"],
                   vecchia_ordering=c["ordering"], seed=c["seed"], cluster_ids=lab if cluster_ids else None, **kw)


def run_case(c, lib=None):
    coords, y, lab, coords_p, lab_p = case_data(c)
    out = dict(name=c["name"])
    gp = model_of(c, coords, lab, lib)
    out["nll"] = float(gp.neg_log_likelihood(np.array(COV_PARS), y))
    gp = model_of(c, coords, lab, lib)
    gp.fit(y, params=dict(trace=False))
    out["cov_pars"] = [float(v) for v in np.asarray(gp.get_cov_pars()).reshape(-1)]
    out["num_it"] = int(gp._get_num_optim_iter())
    out["nll_fit"] = float(gp.get_current_neg_log_likelihood())
    mp = c.get("mp", -1)
    pred = gp.predict(y=y, gp_coords_pred=coords_p, cov_pars=None, predict_var=True, predict_response=True, cluster_ids_pred=lab_p,
                      num_neighbors_pred=mp)
    out["pred_mu"] = [float(v) for v in pred["mu"]]
    out["pred_var"] = [float(v) for v in pred["var"]]
    # latent variances at the fixed parameters (a new cluster: the marginal variance)
    pl = gp.predict(y=y, gp_coords_pred=coords_p, cov_pars=np.array(COV_PARS), predict_var=True, predict_response=False,
                    cluster_ids_pred=lab_p, num_neighbors_pred=mp)
    out["pred_mu_fixed"] = [float(v) for v in pl["mu"]]
    out["pred_var_latent_fixed"] = [float(v) for v in pl["var"]]
    return out


def boost_data(c):
    coords, _, lab, coords_p, lab_p = case_data(c)
    rng = np.random.default_rng(100 + c["seed"])
    n = len(lab)
    X = rng.uniform(-2., 2., size=(n, c["F"]))
    f = np.sin(2. * X[:, 0]) + 0.5 * (X[:, 1] > 0.3) + 0.3 * X[:, 2] ** 2
    shift = {l: rng.normal(0., 1.) for l in c["labels"]}
    b = np.array([np.sin(4. * coords[i, 0]) * np.cos(3. * coords[i, 1]) + 0.5 * shift[lab[i]] for i in range(n)])
    y = f + b + 0.4 * rng.standard_normal(n)
    nv = c["nv"]
    Xv = rng.uniform(-2., 2., size=(nv, c["F"]))
    yv = np.sin(2. * Xv[:, 0]) + 0.4 * rng.standard_normal(nv)
    coords_v = rng.uniform(0., 1., size=(nv, 2))
    lab_v = np.array([c["labels"][k % len(c["labels"])] if k % 5 else NEW_LABEL for k in range(nv)], dtype=np.int32)
    return X, y, coords, lab, Xv, yv, coords_v, lab_v


def run_boost(c, lib=None, train_cov_pars=False, num_it=None, extra=None):
    """trees of num_it iterations (the model string) and the validation metric of every iteration, with the GP for validation; extra:
    more booster parameters (leaves_newton_update, line_search_step_length)"""
    kw = {} if lib is None else dict(_lib=lib)
    X, y, coords, lab, Xv, yv, coords_v, lab_v = boost_data(c)
    params = dict(objective="regression", num_leaves=c["num_leaves"], min_data_in_leaf=20, learning_rate=0.1, max_bin=255, verbose=-1,
                  use_gp_model_for_validation=True, train_gp_model_cov_pars=train_cov_pars, **(extra or {}))
    gp = model_of(c, coords, lab, lib)
    if not train_cov_pars:
        gp.set_optim_params(dict(init_cov_pars=np.array(COV_PARS)))
    gp.set_prediction_data(gp_coords_pred=coords_v, cluster_ids_pred=lab_v)
    dtrain = Dataset(X, y, params=params, free_raw_data=False, **kw)
    dvalid = Dataset(Xv, yv, params=params, reference=dtrain, **kw)
    bst = Booster(params, dtrain, gp_model=gp, **kw)
    bst.add_valid(dvalid, "valid")
    evals = []
    for _ in range(num_it or c["num_it"]):
        bst.update()
        evals.append([[r[0], r[1], r[2]] for r in bst.eval_valid()])
    out = dict(model=bst.model_to_string(), evals=evals,
               cov_pars=[float(v) for v in np.asarray(gp.get_cov_pars()).reshape(-1)])
    return out, bst
