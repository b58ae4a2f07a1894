"""Host-side mirror of the reference's `Dataset` / `Booster` (python-package/gpboost/basic.py:1040-2322, 2323-4170)
for the hot path: dense numerical matrices, `objective=regression`, optional GPModel (GPBoost algorithm).
Same C entry points (`LGBM_*`), bound with ctypes; `_lib` selects the shared library like in GPModel."""
import ctypes

import numpy as np

from .basic import GPBoostError, c_str, _dptr
from .libpath import load_lib

C_API_DTYPE_FLOAT32, C_API_DTYPE_FLOAT64 = 0, 1
C_API_PREDICT_NORMAL, C_API_PREDICT_RAW_SCORE, C_API_PREDICT_LEAF_INDEX, C_API_PREDICT_CONTRIB = 0, 1, 2, 3


def _param_value_str(v):
    if isinstance(v, bool):
        return str(v).lower()
    if isinstance(v, (list, tuple, set)):  # e.g. metric=["l2", "rmse"] -> "l2,rmse" (param_dict_to_str, basic.py)
        return ",".join(str(x) for x in v)
    return v


def param_dict_to_str(params):
    return " ".join("%s=%s" % (k, _param_value_str(v)) for k, v in (params or {}).items())


class Dataset(object):
    def __init__(self, data, label=None, params=None, reference=None, free_raw_data=True, _lib=None):
        """`reference`: the training Dataset whose bin mappers bin this one (validation data, Dataset(..., reference=train_set)).
        `free_raw_data=False` keeps the feature matrix as `self.data` (the library only holds its bins): Booster.predict with a
        GP model needs it to predict the training data."""
        self._LIB = load_lib() if _lib is None else _lib
        self.reference = reference
        self.free_raw_data = free_raw_data
        self.data = None
        data = np.asarray(data)
        # float32 matrices are passed as they are (C_API_DTYPE_FLOAT32), like the reference's package (basic.py: __init_from_np2d)
        dt = np.float32 if data.dtype == np.float32 else np.float64
        data = np.ascontiguousarray(data, dtype=dt)
        if data.ndim != 2:
            raise ValueError("'data' needs to be a 2-D array")
        self.num_data, self.num_feature = data.shape
        self.handle = ctypes.c_void_p()
        self._safe_call(self._LIB.LGBM_DatasetCreateFromMat(
            data.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(C_API_DTYPE_FLOAT32 if dt == np.float32 else C_API_DTYPE_FLOAT64), ctypes.c_int32(self.num_data),
            ctypes.c_int32(self.num_feature), ctypes.c_int(1), c_str(param_dict_to_str(params)),
            None if reference is None else reference.handle, ctypes.byref(self.handle)))
        if not free_raw_data:
            self.data = data
        if label is not None:
            self.set_label(label)

    def _safe_call(self, ret):
        if ret != 0:
            raise GPBoostError(self._LIB.LGBM_GetLastError().decode("utf-8"))

    def set_label(self, label):
        lab = np.ascontiguousarray(np.asarray(label, dtype=np.float32).reshape(-1))  # label_t = float (meta.h:49)
        if lab.shape[0] != self.num_data:
            raise ValueError("Length of label is not same with #data")
        self.label = lab
        self._safe_call(self._LIB.LGBM_DatasetSetField(self.handle, c_str("label"), lab.ctypes.data_as(ctypes.c_void_p),
                                                       ctypes.c_int(lab.shape[0]), ctypes.c_int(C_API_DTYPE_FLOAT32)))

    def __del__(self):
        try:
            if getattr(self, "handle", None) is not None and self.handle.value is not None:
                self._LIB.LGBM_DatasetFree(self.handle)
                self.handle = None
        except Exception:
            pass


class Booster(object):
    def __init__(self, params=None, train_set=None, gp_model=None, model_str=None, model_file=None, _lib=None):
        self._LIB = load_lib() if _lib is None else _lib
        self.train_set, self.gp_model = train_set, gp_model
        self.handle = ctypes.c_void_p()
        self.valid_sets, self.name_valid_sets = [], []
        self._train_data_name = "training"
        self.best_iteration = 0
        self.__eval_names = None
        if model_str is not None or model_file is not None:  # prediction-only booster (Booster(model_file=...), basic.py:2404-2425)
            n_it = ctypes.c_int(0)
            if model_str is not None:
                self._safe_call(self._LIB.LGBM_BoosterLoadModelFromString(c_str(model_str), ctypes.byref(n_it), ctypes.byref(self.handle)))
            else:
                self._safe_call(self._LIB.LGBM_BoosterCreateFromModelfile(c_str(model_file), ctypes.byref(n_it), ctypes.byref(self.handle)))
            return
        params = dict(params or {})
        if gp_model is not None:
            params["has_gp_model"] = True
            self._safe_call(self._LIB.LGBM_GPBoosterCreate(train_set.handle, c_str(param_dict_to_str(params)), gp_model.handle,
                                                           ctypes.byref(self.handle)))
        else:
            self._safe_call(self._LIB.LGBM_BoosterCreate(train_set.handle, c_str(param_dict_to_str(params)), ctypes.byref(self.handle)))

    def _safe_call(self, ret):
        if ret != 0:
            raise GPBoostError(self._LIB.LGBM_GetLastError().decode("utf-8"))

    def update(self):
        """One boosting iteration (Booster.update, basic.py:2846-2905). Returns True when no further split was possible."""
        fin = ctypes.c_int(0)
        self._safe_call(self._LIB.LGBM_BoosterUpdateOneIter(self.handle, ctypes.byref(fin)))
        return fin.value == 1

    def current_iteration(self):
        it = ctypes.c_int(0)
        self._safe_call(self._LIB.LGBM_BoosterGetCurrentIteration(self.handle, ctypes.byref(it)))
        return it.value

    def model_to_string(self, start_iteration=0, num_iteration=-1):
        n = ctypes.c_int64(0)
        buf_len = 1 << 20
        buf = ctypes.create_string_buffer(buf_len)
        self._safe_call(self._LIB.LGBM_BoosterSaveModelToString(self.handle, ctypes.c_int(start_iteration), ctypes.c_int(num_iteration), ctypes.c_int(0),
                                                                ctypes.c_int64(buf_len), ctypes.byref(n), buf))
        if n.value > buf_len:
            buf_len = n.value
            buf = ctypes.create_string_buffer(buf_len)
            self._safe_call(self._LIB.LGBM_BoosterSaveModelToString(self.handle, ctypes.c_int(start_iteration), ctypes.c_int(num_iteration), ctypes.c_int(0),
                                                                    ctypes.c_int64(buf_len), ctypes.byref(n), buf))
        return buf.value.decode("utf-8")

    def save_model(self, filename):
        self._safe_call(self._LIB.LGBM_BoosterSaveModel(self.handle, ctypes.c_int(0), ctypes.c_int(-1), ctypes.c_int(0), c_str(filename)))
        return self

    def inner_predict_train(self):
        """Raw training scores F (Booster.__inner_predict(0), basic.py:3964)."""
        n = ctypes.c_int64(0)
        self._safe_call(self._LIB.LGBM_BoosterGetNumPredict(self.handle, ctypes.c_int(0), ctypes.byref(n)))
        out = np.empty(n.value, dtype=np.float64)
        self._safe_call(self._LIB.LGBM_BoosterGetPredict(self.handle, ctypes.c_int(0), ctypes.byref(n), _dptr(out)))
        return out

    # ---- validation data and metrics (Booster.add_valid / eval_train / eval_valid, basic.py) ---------------------------------
    def set_train_data_name(self, name):
        self._train_data_name = name
        return self

    def add_valid(self, data, name):
        """Add validation data: `data` is a Dataset built with `reference=` the training Dataset."""
        if not isinstance(data, Dataset):
            raise TypeError("Validation data should be Dataset instance, met {}".format(type(data).__name__))
        if data.reference is not self.train_set:
            raise GPBoostError("Add validation data failed, you should use same predictor for these data")
        self._safe_call(self._LIB.LGBM_BoosterAddValidData(self.handle, data.handle))
        self.valid_sets.append(data)
        self.name_valid_sets.append(name)
        return self

    def _eval_names(self):
        if self.__eval_names is None:
            n = ctypes.c_int(0)
            self._safe_call(self._LIB.LGBM_BoosterGetEvalCounts(self.handle, ctypes.byref(n)))
            names = []
            if n.value > 0:
                buf_len = 255
                bufs = [ctypes.create_string_buffer(buf_len) for _ in range(n.value)]
                ptrs = (ctypes.c_char_p * n.value)(*map(ctypes.addressof, bufs))
                out_len, req = ctypes.c_int(0), ctypes.c_size_t(0)
                self._safe_call(self._LIB.LGBM_BoosterGetEvalNames(self.handle, ctypes.c_int(n.value), ctypes.byref(out_len),
                                                                   ctypes.c_size_t(buf_len), ctypes.byref(req), ptrs))
                names = [b.value.decode("utf-8") for b in bufs[:out_len.value]]
            self.__eval_names = names
        return self.__eval_names

    def _inner_eval(self, data_name, data_idx):
        names = self._eval_names()
        if not names:
            return []
        out = np.zeros(len(names), dtype=np.float64)
        n = ctypes.c_int(0)
        self._safe_call(self._LIB.LGBM_BoosterGetEval(self.handle, ctypes.c_int(data_idx), ctypes.byref(n), _dptr(out)))
        if n.value != len(names):
            raise ValueError("Wrong length of eval results")
        # every metric of this build (l2, rmse, l1, test_neg_log_likelihood) is better when lower
        return [(data_name, names[i], float(out[i]), False) for i in range(len(names))]

    def eval_train(self):
        """Metrics on the training data: list of (data_name, eval_name, value, is_higher_better)."""
        return self._inner_eval(self._train_data_name, 0)

    def eval_valid(self):
        """Metrics on every validation set, in the order they were added."""
        out = []
        for i, name in enumerate(self.name_valid_sets):
            out.extend(self._inner_eval(name, i + 1))
        return out

    def inner_predict(self, data_idx):
        """Raw scores of data set `data_idx` (0 training data, k the k-th validation set)."""
        n = ctypes.c_int64(0)
        self._safe_call(self._LIB.LGBM_BoosterGetNumPredict(self.handle, ctypes.c_int(data_idx), ctypes.byref(n)))
        out = np.empty(n.value, dtype=np.float64)
        self._safe_call(self._LIB.LGBM_BoosterGetPredict(self.handle, ctypes.c_int(data_idx), ctypes.byref(n), _dptr(out)))
        return out

    def _predict_for_mat(self, data, predict_type, start_iteration, num_iteration):
        """LGBM_BoosterPredictForMat on a dense matrix (float32 passed as it is, everything else as float64)."""
        data = np.asarray(data)
        dt = np.float32 if data.dtype == np.float32 else np.float64
        data = np.ascontiguousarray(data, dtype=dt)
        if data.ndim != 2:
            raise ValueError("'data' needs to be a 2-D array")
        n = ctypes.c_int64(0)
        self._safe_call(self._LIB.LGBM_BoosterCalcNumPredict(self.handle, ctypes.c_int(data.shape[0]), ctypes.c_int(predict_type),
                                                             ctypes.c_int(start_iteration), ctypes.c_int(num_iteration), ctypes.byref(n)))
        out = np.empty(n.value, dtype=np.float64)
        self._safe_call(self._LIB.LGBM_BoosterPredictForMat(
            self.handle, data.ctypes.data_as(ctypes.c_void_p), ctypes.c_int(C_API_DTYPE_FLOAT32 if dt == np.float32 else C_API_DTYPE_FLOAT64),
            ctypes.c_int32(data.shape[0]), ctypes.c_int32(data.shape[1]), ctypes.c_int(1), ctypes.c_int(predict_type),
            ctypes.c_int(start_iteration), ctypes.c_int(num_iteration), c_str(""), ctypes.byref(n), _dptr(out)))
        if n.value != out.shape[0]:
            raise ValueError("Wrong length for predict results")
        if predict_type == C_API_PREDICT_LEAF_INDEX:
            return out.astype(np.int32).reshape(data.shape[0], out.shape[0] // data.shape[0])
        return out

    def predict(self, data, start_iteration=0, num_iteration=None, raw_score=None, pred_leaf=False, pred_latent=False, gp_coords_pred=None,
                predict_var=False, cov_pars=None, ignore_gp_model=False, offset_pred=None, num_neighbors_pred=-1, pred_contrib=False,
                predict_cov_mat=False, sample_posterior=False, cluster_ids_pred=None):
        """Prediction at new data (Booster.predict, basic.py:3376-3802). Without a `gp_model` (or with `ignore_gp_model=True`): the
        tree ensemble's scores, or with `pred_leaf=True` the (nrow, trees) leaf indices. With a Gaussian `gp_model`: the reference's
        dict — `pred_latent=True`: fixed_effect, random_effect_mean, random_effect_cov (the variances, with `predict_var`);
        `pred_latent=False`: response_mean, response_var. The GP predicts from the residual label - F(X_train), so the training
        Dataset must have been built with `free_raw_data=False`. `num_iteration=None` uses `best_iteration`. An explicit `raw_score`
        (an argument the reference has discontinued) asks for the tree ensemble's scores alone, as it always has here, also with a
        `gp_model`."""
        if pred_contrib:
            raise GPBoostError("Feature contributions (pred_contrib) are not supported by this build")
        if predict_cov_mat or sample_posterior:
            raise GPBoostError("Predictive covariance matrices (predict_cov_mat) and posterior samples (sample_posterior) are not supported "
                               "by this build")
        if num_iteration is None:  # basic.py:3623-3627
            num_iteration = self.best_iteration if start_iteration <= 0 else -1
        if self.gp_model is None or ignore_gp_model or raw_score is not None:
            ptype = C_API_PREDICT_LEAF_INDEX if pred_leaf else (C_API_PREDICT_NORMAL if raw_score is False else C_API_PREDICT_RAW_SCORE)
            return self._predict_for_mat(data, ptype, start_iteration, num_iteration)
        if pred_leaf:
            raise GPBoostError("pred_leaf with a gp_model is not supported by this build: set ignore_gp_model=True for the leaf indices")
        if self.train_set is None or getattr(self.train_set, "data", None) is None:
            raise GPBoostError("Cannot make predictions for Gaussian process. Set free_raw_data = False when you construct the Dataset")
        if self.gp_model._get_likelihood_name() != "gaussian":
            raise GPBoostError("Prediction with a gp_model is only supported for the gaussian likelihood by this build (likelihood: %s)"
                               % self.gp_model._get_likelihood_name())
        if gp_coords_pred is None:
            raise GPBoostError("'gp_coords_pred' is needed for the prediction with a gp_model")
        # basic.py:3646-3700: the GP predicts from the residual of the training data under the same trees
        fixed_effect_train = self._predict_for_mat(self.train_set.data, C_API_PREDICT_RAW_SCORE, start_iteration, num_iteration)
        residual = self.train_set.label - fixed_effect_train
        re_pred = self.gp_model.predict(y=residual, gp_coords_pred=gp_coords_pred, cov_pars=cov_pars, predict_var=predict_var,
                                        predict_response=not pred_latent, num_neighbors_pred=num_neighbors_pred,
                                        cluster_ids_pred=cluster_ids_pred)
        fixed_effect = self._predict_for_mat(data, C_API_PREDICT_RAW_SCORE, start_iteration, num_iteration)
        if len(fixed_effect) != len(re_pred["mu"]):
            raise GPBoostError("Number of data points in fixed effect (tree ensemble) and random effect are not equal")
        if offset_pred is not None:
            offset_pred = np.asarray(offset_pred, dtype=np.float64).reshape(-1)
            if len(fixed_effect) != len(offset_pred):
                raise GPBoostError("Number of data points in fixed effect (tree ensemble) and 'offset_pred' are not equal")
            fixed_effect = fixed_effect + offset_pred
        out = {"fixed_effect": None, "random_effect_mean": None, "random_effect_cov": None, "response_mean": None, "response_var": None}
        if pred_latent:
            out["fixed_effect"] = fixed_effect
            out["random_effect_mean"] = re_pred["mu"]
            out["random_effect_cov"] = re_pred["var"] if predict_var else None
        else:
            out["response_mean"] = re_pred["mu"] + fixed_effect
            out["response_var"] = re_pred["var"] if predict_var else None
        return out

    def __del__(self):
        try:
            if getattr(self, "handle", None) is not None and self.handle.value is not None:
                self._LIB.LGBM_BoosterFree(self.handle)
                self.handle = None
        except Exception:
            pass


def parse_model_string(s):
    """Trees of a LightGBM/GPBoost text model -> list of dicts of numpy arrays (io/gbdt_model_text.cpp, Tree::ToString)."""
    trees = []
    cur = None
    for line in s.splitlines():
        if line.startswith("Tree="):
            cur = {}
            trees.append(cur)
        elif cur is not None and "=" in line:
            k, v = line.split("=", 1)
            if k in ("split_feature", "left_child", "right_child", "leaf_count", "internal_count", "decision_type"):
                cur[k] = np.array([int(x) for x in v.split()], dtype=np.int64)
            elif k in ("threshold", "leaf_value", "split_gain", "internal_value", "leaf_weight", "internal_weight"):
                cur[k] = np.array([float(x) for x in v.split()], dtype=np.float64)
            elif k in ("num_leaves", "num_cat"):
                cur[k] = int(v)
            elif k == "shrinkage":
                cur[k] = float(v)
        elif line.startswith("end of trees"):
            break
    return trees
