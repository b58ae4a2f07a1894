"""`train` of the reference's Python package (python-package/gpboost/engine.py:26-400) for this build's Booster: boosting with
validation data, evaluation after every iteration, `evals_result` and early stopping with the rule of `callback.early_stopping`
(callback.py:146-237). Early stopping does not roll the booster back: it records `best_iteration` (1-based), like the reference."""
import collections
import copy

from .booster import Booster, Dataset

_ES_ALIASES = ("early_stopping_round", "early_stopping_rounds", "early_stopping", "n_iter_no_change")
_NUM_IT_ALIASES = ("num_iterations", "num_iteration", "n_iter", "num_tree", "num_trees", "num_round", "num_rounds",
                   "num_boost_round", "n_estimators")


class EarlyStopException(Exception):
    def __init__(self, best_iteration, best_score):
        super().__init__()
        self.best_iteration = best_iteration
        self.best_score = best_score


def _early_stopping(stopping_rounds, first_metric_only, train_data_name):
    """callback.early_stopping (callback.py:146-237): per-metric best score; the training data only ends the last round"""
    best_score, best_iter, best_score_list, higher_better = [], [], [], []
    first_metric = [""]

    def _init(results):
        if not results:
            raise ValueError("For early stopping, at least one dataset and eval metric is required for evaluation")
        first_metric[0] = results[0][1].split(" ")[-1]
        for r in results:
            best_iter.append(0)
            best_score_list.append(None)
            higher_better.append(bool(r[3]))
            best_score.append(float("-inf") if r[3] else float("inf"))

    def _callback(iteration, end_iteration, results):
        if not higher_better:
            _init(results)
        for i in range(len(results)):
            score = results[i][2]
            better = score > best_score[i] if higher_better[i] else score < best_score[i]
            if best_score_list[i] is None or better:
                best_score[i] = score
                best_iter[i] = iteration
                best_score_list[i] = results
            name_split = results[i][1].split(" ")
            if first_metric_only and first_metric[0] != name_split[-1]:
                continue
            if results[i][0] == train_data_name:
                if iteration == end_iteration - 1:
                    raise EarlyStopException(best_iter[i], best_score_list[i])
                continue
            if iteration - best_iter[i] >= stopping_rounds:
                raise EarlyStopException(best_iter[i], best_score_list[i])
            if iteration == end_iteration - 1:
                raise EarlyStopException(best_iter[i], best_score_list[i])
    return _callback


def train(params, train_set, num_boost_round=100, valid_sets=None, valid_names=None, gp_model=None, use_gp_model_for_validation=True,
          train_gp_model_cov_pars=True, early_stopping_rounds=None, evals_result=None):
    """Boost `num_boost_round` trees on `train_set` (optionally with a GPModel), evaluating the metrics of `params["metric"]` on
    `valid_sets` after every iteration. With `early_stopping_rounds`, training stops once no metric of a validation set has improved in
    that many rounds; `booster.best_iteration` (1-based) and `booster.best_score` record the best round. `evals_result` (a dict) receives
    every round's values, {data_name: {eval_name: [values]}}."""
    params = copy.deepcopy(params or {})
    for alias in _NUM_IT_ALIASES:
        if alias in params:
            num_boost_round = params.pop(alias)
    for alias in _ES_ALIASES:
        if alias in params:
            early_stopping_rounds = params.pop(alias)
    first_metric_only = bool(params.get("first_metric_only", False))
    if num_boost_round <= 0:
        raise ValueError("num_boost_round should be greater than zero.")
    if not isinstance(train_set, Dataset):
        raise TypeError("Training only accepts Dataset object")
    is_valid_contain_train = False
    train_data_name = "training"
    reduced_valid_sets, name_valid_sets = [], []
    if valid_sets is not None:
        if isinstance(valid_sets, Dataset):
            valid_sets = [valid_sets]
        if isinstance(valid_names, str):
            valid_names = [valid_names]
        for i, valid_data in enumerate(valid_sets):
            if valid_data is train_set:
                is_valid_contain_train = True
                if valid_names is not None:
                    train_data_name = valid_names[i]
                continue
            if not isinstance(valid_data, Dataset):
                raise TypeError("Training only accepts Dataset object")
            reduced_valid_sets.append(valid_data)
            name_valid_sets.append(valid_names[i] if valid_names is not None and len(valid_names) > i else "valid_" + str(i))
    if gp_model is not None:
        if getattr(gp_model, "has_covariates", False):
            raise ValueError("The 'gp_model' cannot have covariates 'X' (a linear predictor) in the GPBoost algorithm.")
        if use_gp_model_for_validation and len(reduced_valid_sets) > 1:
            raise ValueError("Can use only one validation set when use_gp_model_for_validation = True")
        if not is_valid_contain_train and use_gp_model_for_validation and len(reduced_valid_sets) > 0 and \
                not gp_model.prediction_data_is_set:
            raise ValueError("Prediction data for 'gp_model' has not been set. "
                             "This needs to be set prior to trainig when having a validation set and 'use_gp_model_for_validation=True'. "
                             "Either call 'gp_model.set_prediction_data(...)' first or use 'use_gp_model_for_validation=False'.")
        params["use_gp_model_for_validation"] = use_gp_model_for_validation
        params["train_gp_model_cov_pars"] = train_gp_model_cov_pars
        if is_valid_contain_train and len(reduced_valid_sets) == 0 and params.get("metric") is None:
            params["metric"] = "neg_log_likelihood"  # engine.py:291-296 (Gaussian likelihood)
    if early_stopping_rounds is not None and early_stopping_rounds > 0:
        params["early_stopping_round"] = early_stopping_rounds
    booster = Booster(params=params, train_set=train_set, gp_model=gp_model, _lib=train_set._LIB)
    if is_valid_contain_train:
        booster.set_train_data_name(train_data_name)
    for valid_set, name in zip(reduced_valid_sets, name_valid_sets):
        booster.add_valid(valid_set, name)
    booster.best_iteration = 0
    es = None
    if early_stopping_rounds is not None and early_stopping_rounds > 0:
        es = _early_stopping(early_stopping_rounds, first_metric_only, train_data_name)
    if evals_result is not None:
        if not isinstance(evals_result, dict):
            raise TypeError("eval_result should be a dictionary")
        evals_result.clear()
    results = []
    for i in range(num_boost_round):
        booster.update()
        results = []
        if valid_sets is not None:
            if is_valid_contain_train:
                results.extend(booster.eval_train())
            results.extend(booster.eval_valid())
        if evals_result is not None:  # callback.record_evaluation (order 20, before early stopping)
            for data_name, eval_name, value, _ in results:
                evals_result.setdefault(data_name, collections.OrderedDict()).setdefault(eval_name, []).append(value)
        if es is not None:
            try:
                es(i, num_boost_round, results)
            except EarlyStopException as stop:
                booster.best_iteration = stop.best_iteration + 1
                results = stop.best_score
                break
    booster.best_score = collections.defaultdict(collections.OrderedDict)
    for data_name, eval_name, score, _ in results:
        booster.best_score[data_name][eval_name] = score
    return booster
