"""Cases of the validation-data goldens (tests/golden/make_validation_golden.py) and the code that runs one case through the shared
frontend (gpboost_b200.booster / GPModel / train), on this build's library or, with `lib`, on the unmodified reference library."""
import numpy as np

from gpboost_b200 import GPModel
from gpboost_b200.booster import Booster, Dataset

NUM_IT = 10

CASES = [
    # plain boosting, three metrics, two validation sets
    dict(name="plain_two_valid", n=2000, nv=[500, 400], F=6, seed=1, num_leaves=15, metric="l2,rmse,l1", gp=None),
    # the training data passed as a validation set (data index 0) next to a real one
    dict(name="train_as_valid", n=1500, nv=[300], F=5, seed=2, num_leaves=8, metric="mse,l2_root,mae", gp=None, train_as_valid=True),
    # validation data added after 5 iterations: the trees trained so far are replayed
    dict(name="late_add_replay", n=1800, nv=[600], F=6, seed=3, num_leaves=31, metric="l2", gp=None, add_after=5),
    # test_neg_log_likelihood without a GP: the training residual variance
    dict(name="plain_test_nll", n=1200, nv=[400], F=4, seed=4, num_leaves=10, metric="l2,test_neg_log_likelihood", gp=None),
    # GPBoost with a Vecchia GP at fixed covariance parameters
    dict(name="vecchia_default_gpval", n=1500, nv=[400], F=4, seed=5, num_leaves=10, metric=None, gp="vecchia", use_gp=True),
    dict(name="vecchia_default_nogpval", n=1500, nv=[400], F=4, seed=5, num_leaves=10, metric=None, gp="vecchia", use_gp=False),
    dict(name="vecchia_l2_gpval", n=1500, nv=[400], F=4, seed=6, num_leaves=10, metric="l2", gp="vecchia", use_gp=True),
    # grouped random effect validated on the tree scores
    dict(name="grouped_nogpval", n=1500, nv=[400], F=4, seed=7, num_leaves=10, metric="l2,test_neg_log_likelihood", gp="grouped",
         use_gp=False),
]
# an early-stopping run that stops before num_boost_round (gpboost_b200.train / gpb.train)
ES_CASE = dict(name="early_stopping", n=1500, nv=[500], F=5, seed=8, num_leaves=31, metric="l2,l1", learning_rate=0.3,
               num_boost_round=60, early_stopping_rounds=3)

COV_PARS = [0.3, 1.0, 0.15]       # error variance, GP variance, range (Vecchia, exponential)
COV_PARS_GROUPED = [0.3, 0.5]    # error variance, group variance


def case_data(c):
    """X, y, coords, groups of the training data followed by the validation sets: list of (X, y, coords, groups)"""
    rng = np.random.default_rng(c["seed"])
    sizes = [c["n"]] + list(c["nv"])
    out = []
    for m in sizes:
        X = rng.uniform(-2., 2., size=(m, c["F"]))
        coords = rng.uniform(0., 1., size=(m, 2))
        groups = rng.integers(0, 30, size=m)
        f = np.sin(2. * X[:, 0]) + 0.5 * (X[:, 1] > 0.3) + 0.3 * X[:, 2] ** 2
        b = np.sin(4. * coords[:, 0]) * np.cos(3. * coords[:, 1]) + 0.05 * groups / 30.
        y = f + b + 0.4 * rng.standard_normal(m)
        out.append((X, y, coords, groups))
    return out


def params_of(c):
    p = dict(objective="regression", num_leaves=c["num_leaves"], min_data_in_leaf=20, learning_rate=c.get("learning_rate", 0.1),
             max_bin=255, verbose=-1)
    if c.get("metric") is not None:
        p["metric"] = c["metric"]
    if c.get("gp") is not None:
        p["use_gp_model_for_validation"] = c["use_gp"]
        p["train_gp_model_cov_pars"] = False
    return p


def gp_model_of(c, data, lib=None):
    kw = {} if lib is None else dict(_lib=lib)
    X, y, coords, groups = data[0]
    if c.get("gp") == "vecchia":
        gp = GPModel(gp_coords=coords, cov_function="exponential", gp_approx="vecchia", num_neighbors=10, vecchia_ordering="random",
                     seed=c["seed"], **kw)
        gp.set_optim_params(dict(init_cov_pars=np.array(COV_PARS)))
        gp.set_prediction_data(gp_coords_pred=data[1][2], num_neighbors_pred=20)
        return gp
    if c.get("gp") == "grouped":
        gp = GPModel(group_data=groups, **kw)
        gp.set_optim_params(dict(init_cov_pars=np.array(COV_PARS_GROUPED)))
        return gp
    return None


def metric_names(c):
    m = c.get("metric")
    if m is None:
        return ["test_neg_log_likelihood"] if c.get("gp") else ["l2"]
    return m.split(",")


def needs_train_scores(c):
    return not (c.get("gp") and c.get("use_gp")) and "test_neg_log_likelihood" in metric_names(c)


def run_case(c, lib=None, record_scores=True):
    """per iteration: the evaluation list; at the end the raw validation scores (GetPredict) of every validation set"""
    kw = {} if lib is None else dict(_lib=lib)
    data = case_data(c)
    params = params_of(c)
    X, y = data[0][0], data[0][1]
    dtrain = Dataset(X, y, params=params, **kw)
    dvalid = [Dataset(Xv, yv, params=params, reference=dtrain, **kw) for (Xv, yv, _, _) in data[1:]]
    gp = gp_model_of(c, data, lib)
    bst = Booster(params, dtrain, gp_model=gp, **kw)
    if c.get("train_as_valid"):
        bst.set_train_data_name("training")
    add_after = c.get("add_after", 0)
    evals = []

    def add_all():
        for i, dv in enumerate(dvalid):
            bst.add_valid(dv, "valid_%d" % i)

    if add_after == 0:
        add_all()
    for it in range(NUM_IT):
        if it == add_after and add_after > 0:
            add_all()
        bst.update()
        if it + 1 >= max(add_after, 1):
            res = (bst.eval_train() if c.get("train_as_valid") else []) + bst.eval_valid()
            evals.append([[r[0], r[1], r[2]] for r in res])
    out = dict(evals=evals, eval_names=bst._eval_names())
    if record_scores:
        out["valid_scores"] = [[float(v).hex() for v in bst.inner_predict(k + 1)] for k in range(len(dvalid))]
        if needs_train_scores(c):  # the residual variance of test_neg_log_likelihood without the GP
            out["train_scores"] = [float(v).hex() for v in bst.inner_predict(0)]
    return out, bst, data, gp


def run_es_case(c, lib=None):
    from gpboost_b200 import train
    kw = {} if lib is None else dict(_lib=lib)
    data = case_data(c)
    params = params_of(c)
    dtrain = Dataset(data[0][0], data[0][1], params=params, **kw)
    dvalid = Dataset(data[1][0], data[1][1], params=params, reference=dtrain, **kw)
    evals_result = {}
    bst = train(params, dtrain, num_boost_round=c["num_boost_round"], valid_sets=[dvalid], valid_names=["valid"],
                early_stopping_rounds=c["early_stopping_rounds"], evals_result=evals_result)
    return dict(best_iteration=bst.best_iteration, evals_result={k: dict(v) for k, v in evals_result.items()},
                num_trees=bst.current_iteration())
