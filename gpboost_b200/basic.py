"""Host-side mirror of the reference's Python `GPModel` (python-package/gpboost/basic.py:4172-7122) for the
hot-path configurations: same constructor arguments, method names, argument meaning and error behaviour, bound
with ctypes to the same C API (`GPB_*`). The class takes the shared library as an optional argument so that the
parity tests can drive the UNMODIFIED reference build (oracle/_ref/lib_gpboost.so) and this repository's
`lib_gpboost_b200.so` through identical calls.
"""
import ctypes
import numpy as np

from .libpath import load_lib


class GPBoostError(Exception):
    """Error raised by the C API (mirrors gpboost.basic.GPBoostError)."""


def c_str(s):
    return ctypes.c_char_p(s.encode("utf-8"))


def _as_1d(a, name, n=None):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(-1))
    if n is not None and a.shape[0] != n:
        raise ValueError("Incorrect number of data points in '%s'" % name)
    return a


def _dptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


# defaults of GPModel.params (python-package/gpboost/basic.py:4725-4760): -999 / -1 = "use the C++ default"
_DEFAULT_PARAMS = {
    "maxit": 1000, "delta_rel_conv": -999., "init_coef": None, "lr_coef": 0.1, "lr_cov": -999.,
    "use_nesterov_acc": True, "acc_rate_coef": 0.5, "acc_rate_cov": 0.5, "nesterov_schedule_version": 0,
    "momentum_offset": 2, "trace": False, "convergence_criterion": "relative_change_in_log_likelihood",
    "std_dev": False, "init_cov_pars": None, "optimizer_cov": None, "optimizer_coef": None,
    "cg_max_num_it": 1000, "cg_max_num_it_tridiag": 1000, "cg_delta_conv": 1e-2, "num_rand_vec_trace": 50,
    "reuse_rand_vec_trace": True, "cg_preconditioner_type": None, "seed_rand_vec_trace": 1,
    "fitc_piv_chol_preconditioner_rank": -999, "init_aux_pars": None, "estimate_aux_pars": True,
    "init_coef_aux_pars_from_iid_model": True, "estimate_cov_par_index": None, "m_lbfgs": -999,
    "delta_conv_mode_finding": -999.,
}


class GPModel(object):
    """Gaussian process / mixed effects model (hot-path subset of gpboost.GPModel)."""

    def __init__(self, likelihood="gaussian", group_data=None, gp_coords=None, cov_function="matern",
                 cov_fct_shape=1.5, gp_approx="none", num_parallel_threads=None, GPU_use=False,
                 matrix_inversion_method="default", weights=None, num_neighbors=None, vecchia_ordering="random",
                 seed=0, cluster_ids=None, _lib=None):
        self._LIB = load_lib() if _lib is None else _lib
        self.handle = ctypes.c_void_p()
        if gp_coords is None and group_data is None:
            raise ValueError("Both 'group_data' and 'gp_coords' are None. Provide at least one of them")
        if weights is not None:
            raise ValueError("'weights' are not supported by gpboost_b200.GPModel yet")
        self.num_group_re, self.num_gp, self.dim_coords = 0, 0, 0
        group_c, coords_ptr = None, None
        if group_data is not None:
            group_data = np.asarray(group_data)
            if group_data.ndim == 1:
                group_data = group_data.reshape(-1, 1)
            self.num_data, self.num_group_re = group_data.shape
            # labels as NUL-terminated strings, column-major (string_array_c_str, basic.py:224-226, :4922-4923)
            self._group_bytes = "\0".join(str(v) for v in group_data.flatten(order="F")).encode("utf-8") + b"\0"
            group_c = ctypes.c_char_p(self._group_bytes)
        if gp_coords is not None:
            gp_coords = np.asarray(gp_coords, dtype=np.float64)
            if gp_coords.ndim == 1:
                gp_coords = gp_coords.reshape(-1, 1)
            if gp_coords.ndim != 2:
                raise ValueError("'gp_coords' needs to be a 2-D array")
            self.num_data, self.dim_coords = gp_coords.shape
            self.num_gp = 1
        self.likelihood = likelihood
        self.cov_function, self.cov_fct_shape = cov_function, float(cov_fct_shape)
        self.gp_approx, self.vecchia_ordering, self.seed = gp_approx, vecchia_ordering, int(seed)
        self.num_neighbors = -1 if num_neighbors is None else int(num_neighbors)
        self.num_parallel_threads = -1 if num_parallel_threads is None else int(num_parallel_threads)
        gauss = likelihood in ("gaussian", "regression")
        # GP parameter names as in the reference package (basic.py:5040-5070): one range per coordinate for the ARD kernels, a time and
        # a space range for the space-time kernel
        gp_names = ["GP_var", "GP_range"]
        if cov_function in ("matern_space_time", "exponential_space_time", "Matern_space_time"):
            gp_names = ["GP_var", "GP_range_time", "GP_range_space"]
        elif cov_function in ("matern_ard", "gaussian_ard", "exponential_ard", "Matern_ard"):
            gp_names = ["GP_var"] + ["GP_range_" + str(i + 1) for i in range(self.dim_coords)]
        self.num_cov_pars = (1 if gauss else 0) + self.num_group_re + (len(gp_names) if self.num_gp else 0)
        self.cov_par_names = (["Error_term"] if gauss else []) + ["Group_%d" % (k + 1) for k in range(self.num_group_re)] + \
            (gp_names if self.num_gp else [])
        self.params = dict(_DEFAULT_PARAMS)
        self.num_coef = 0
        self.num_covariates = 0
        self.has_covariates = False
        if self.num_gp:
            self._coords_c = np.asfortranarray(gp_coords)  # column-major, gp_coords_data[j*num_data+i]
            coords_ptr = _dptr(self._coords_c)
        cluster_c = None
        if cluster_ids is not None:
            cl = np.ascontiguousarray(np.asarray(cluster_ids).astype(np.int32))
            if cl.shape[0] != self.num_data:
                raise ValueError("Incorrect number of data points in 'cluster_ids'")
            cluster_c = cl.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        self._safe_call(self._LIB.GPB_CreateREModel(
            ctypes.c_int32(self.num_data), cluster_c, group_c, ctypes.c_int32(self.num_group_re), None, None, ctypes.c_int32(0), None,
            ctypes.c_int32(self.num_gp), coords_ptr, ctypes.c_int(self.dim_coords), None, ctypes.c_int32(0),
            c_str(cov_function), ctypes.c_double(self.cov_fct_shape), c_str(gp_approx), ctypes.c_double(1.),
            ctypes.c_double(1.), ctypes.c_int(self.num_neighbors), c_str(vecchia_ordering), ctypes.c_int(-1),
            ctypes.c_double(1.), c_str("kmeans++"), c_str(likelihood), ctypes.c_double(-999.),
            c_str(matrix_inversion_method), ctypes.c_int(self.seed), ctypes.c_int(self.num_parallel_threads),
            ctypes.c_bool(bool(GPU_use)), ctypes.c_bool(False), None, ctypes.c_double(1.), ctypes.byref(self.handle)))

    # ------------------------------------------------------------------------------------------------
    def _safe_call(self, ret):
        if ret != 0:
            raise GPBoostError(self._LIB.LGBM_GetLastError().decode("utf-8"))

    def __del__(self):
        try:
            if getattr(self, "handle", None) is not None and self.handle.value is not None:
                self._LIB.GPB_REModelFree(self.handle)
                self.handle = None
        except Exception:
            pass

    def set_optim_params(self, params):
        """Set parameters for estimation / optimisation (GPModel.set_optim_params, basic.py:5702-5925)."""
        if params is not None:
            for k, v in params.items():
                if k in ("optimizer_cov", "init_cov_pars", "maxit", "delta_rel_conv", "lr_cov", "trace",
                         "convergence_criterion", "m_lbfgs", "estimate_cov_par_index", "std_dev", "cg_max_num_it",
                         "cg_max_num_it_tridiag", "cg_delta_conv", "num_rand_vec_trace", "seed_rand_vec_trace",
                         "cg_preconditioner_type", "delta_conv_mode_finding", "optimizer_coef", "reuse_rand_vec_trace",
                         "init_coef_aux_pars_from_iid_model"):
                    self.params[k] = v
                elif k == "init_coef":
                    if v is None:
                        self.params[k] = None
                        continue
                    v = _as_1d(v, "init_coef")
                    if self.num_coef == 0:  # basic.py:5335-5344
                        self.num_coef = v.shape[0]
                    if v.shape[0] != self.num_coef:
                        raise ValueError("params['init_coef'] does not contain the correct number of parameters")
                    self.params[k] = v
                else:
                    raise ValueError("Unknown or unsupported parameter: %s" % k)
        init_c = None
        if self.params["init_cov_pars"] is not None:
            self._init_cov = _as_1d(self.params["init_cov_pars"], "init_cov_pars", self.num_cov_pars)
            init_c = _dptr(self._init_cov)
        opt_c = c_str(self.params["optimizer_cov"]) if self.params["optimizer_cov"] is not None else None
        init_coef_c = None
        if self.params["init_coef"] is not None:
            self._init_coef = _as_1d(self.params["init_coef"], "init_coef", self.num_coef)
            init_coef_c = _dptr(self._init_coef)
        opt_coef_c = c_str(self.params["optimizer_coef"]) if self.params["optimizer_coef"] is not None else None
        est = self.params["estimate_cov_par_index"]
        est = np.full(self.num_cov_pars, -1, dtype=np.int32) if est is None else np.ascontiguousarray(est, dtype=np.int32)
        self._safe_call(self._LIB.GPB_SetOptimConfig(
            self.handle, init_c, ctypes.c_double(self.params["lr_cov"]), ctypes.c_double(self.params["acc_rate_cov"]),
            ctypes.c_int(self.params["maxit"]), ctypes.c_double(self.params["delta_rel_conv"]),
            ctypes.c_bool(self.params["use_nesterov_acc"]), ctypes.c_int(self.params["nesterov_schedule_version"]),
            ctypes.c_bool(self.params["trace"]), opt_c, ctypes.c_int(self.params["momentum_offset"]),
            c_str(self.params["convergence_criterion"]), ctypes.c_int(self.num_coef), init_coef_c,
            ctypes.c_double(self.params["lr_coef"]), ctypes.c_double(self.params["acc_rate_coef"]), opt_coef_c,
            ctypes.c_int(self.params["cg_max_num_it"]), ctypes.c_int(self.params["cg_max_num_it_tridiag"]),
            ctypes.c_double(self.params["cg_delta_conv"]), ctypes.c_int(self.params["num_rand_vec_trace"]),
            ctypes.c_bool(self.params["reuse_rand_vec_trace"]),
            c_str(self.params["cg_preconditioner_type"]) if self.params.get("cg_preconditioner_type") else None,
            ctypes.c_int(self.params["seed_rand_vec_trace"]),
            ctypes.c_int(self.params["fitc_piv_chol_preconditioner_rank"]), None,
            ctypes.c_bool(self.params["estimate_aux_pars"]), ctypes.c_bool(self.params["init_coef_aux_pars_from_iid_model"]),
            est.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), ctypes.c_int(self.params["m_lbfgs"]),
            ctypes.c_double(self.params["delta_conv_mode_finding"])))
        return self

    def fit(self, y, X=None, params=None, offset=None, fixed_effects=None):
        """Find the covariance parameters that minimise the negative log-likelihood (GPModel.fit, basic.py:5394); with covariates
        `X` (n x p) also the linear regression coefficients, profiled out by GLS in every evaluation (basic.py:5590-5627)."""
        if offset is None:
            offset = fixed_effects
        y = _as_1d(y, "y", self.num_data)
        X_c = None
        if X is not None:
            X = np.asarray(X, dtype=np.float64)
            if X.ndim == 1:
                X = X.reshape(-1, 1)
            if X.ndim != 2 or X.shape[0] != self.num_data:
                raise GPBoostError("Incorrect number of data points in X")
            self.num_covariates = X.shape[1]
            self.num_coef = self.num_covariates
            self._X_c = np.ascontiguousarray(X.flatten(order="F"))  # column-major, covariate_data[j*num_data+i]
            X_c = _dptr(self._X_c)
        self.set_optim_params(params)
        off_c = None
        if offset is not None:
            offset = _as_1d(offset, "offset", self.num_data)
            off_c = _dptr(offset)
        if X is None:
            self._safe_call(self._LIB.GPB_OptimCovPar(self.handle, _dptr(y), off_c))
        else:
            self._safe_call(self._LIB.GPB_OptimLinRegrCoefCovPar(self.handle, _dptr(y), X_c, ctypes.c_int(self.num_covariates), off_c))
        self.has_covariates = X is not None
        return self

    def get_coef(self, std_err=False):
        """Linear regression coefficients of the last fit with covariates (GPModel.get_coef, basic.py:6010-6050)."""
        out = np.zeros(self.num_coef, dtype=np.float64)
        self._safe_call(self._LIB.GPB_GetCoef(self.handle, _dptr(out), ctypes.c_bool(bool(std_err))))
        return out

    def neg_log_likelihood(self, cov_pars, y, fixed_effects=None):
        """Evaluate the negative log-likelihood at `cov_pars` on the original scale (basic.py:5636-5700)."""
        y = _as_1d(y, "y", self.num_data)
        cov_pars = _as_1d(cov_pars, "cov_pars")
        if cov_pars.shape[0] != self.num_cov_pars:
            raise ValueError("'cov_pars' does not contain the correct number of parameters")
        fe_c = None
        if fixed_effects is not None:
            fixed_effects = _as_1d(fixed_effects, "fixed_effects", self.num_data)
            fe_c = _dptr(fixed_effects)
        negll = ctypes.c_double(0)
        self._safe_call(self._LIB.GPB_EvalNegLogLikelihood(self.handle, _dptr(y), _dptr(cov_pars), fe_c, ctypes.byref(negll)))
        return negll.value

    def get_cov_pars(self, std_err=False, format_pandas=False):
        """Covariance parameters on the original scale (GPModel.get_cov_pars, basic.py:5964-6008). With `std_err` and a model
        for which the library computes them, a 2 x num_cov_pars array: the parameters ("Param.") and their standard errors
        ("Std. err."); otherwise the parameters alone."""
        if std_err and not self._can_calculate_standard_errors_cov_pars():
            std_err = False
        k = self.num_cov_pars
        out = np.zeros(2 * k if std_err else k, dtype=np.float64)
        self._safe_call(self._LIB.GPB_GetCovPar(self.handle, _dptr(out), ctypes.c_bool(std_err)))
        if std_err:
            out = np.vstack((out[:k], out[k:]))
        if format_pandas:
            import pandas as pd
            if std_err:
                return pd.DataFrame(out, columns=self.cov_par_names, index=["Param.", "Std. err."])
            return pd.DataFrame(out.reshape(1, -1), columns=self.cov_par_names, index=["Param."])
        return out

    def _can_calculate_standard_errors_cov_pars(self):
        out = ctypes.c_int(0)
        self._safe_call(self._LIB.GPB_CanCalculateStandardErrorsCovPars(self.handle, ctypes.byref(out)))
        return bool(out.value)

    def laplace_info(self):
        """gpboost_b200 extension: (negll, Newton its, CG its, SLQ its, log det(Sigma W + I), objective at the mode)."""
        out = np.zeros(6)
        self._safe_call(self._LIB.GPB200_GetLaplaceInfo(self.handle, _dptr(out)))
        return out

    def laplace_mode(self):
        """gpboost_b200 extension: posterior mode of the latent process (original data order)."""
        out = np.zeros(self.num_data)
        self._safe_call(self._LIB.GPB200_GetLaplaceMode(self.handle, _dptr(out)))
        return out

    def get_current_neg_log_likelihood(self):
        negll = ctypes.c_double(0)
        self._safe_call(self._LIB.GPB_GetCurrentNegLogLikelihood(self.handle, ctypes.byref(negll)))
        return negll.value

    def _get_num_optim_iter(self):
        it = ctypes.c_int(0)
        self._safe_call(self._LIB.GPB_GetNumIt(self.handle, ctypes.byref(it)))
        return it.value

    def _get_num_neighbor_searches(self):
        """searches of the Vecchia neighbour sets in the scaled space of an anisotropic kernel (GPB200_GetNumNeighborSearches)"""
        c = ctypes.c_int(0)
        self._safe_call(self._LIB.GPB200_GetNumNeighborSearches(self.handle, ctypes.byref(c)))
        return c.value

    def _get_likelihood_name(self):
        buf = ctypes.create_string_buffer(256)
        n = ctypes.c_int(0)
        self._safe_call(self._LIB.GPB_GetLikelihoodName(self.handle, buf, ctypes.byref(n)))
        return buf.value.decode()

    def predict(self, y, gp_coords_pred, cov_pars, predict_var=False, predict_response=True, vecchia_pred_type=None,
                num_neighbors_pred=-1, X_pred=None, cluster_ids_pred=None):
        """Predictive mean (and variance) at new locations (GPModel.predict, basic.py:6168-6520 -> GPB_SetPredictionData,
        GPB_PredictREModel), GP part only. Returns dict(mu, var). This library does not export the prediction entries
        yet (SURVEY §8 f1); with `_lib` = the reference library this produces the golden vectors for them."""
        if not hasattr(self._LIB, "GPB_PredictREModel"):
            raise GPBoostError("GPB_PredictREModel is not exported by this library (prediction with the GP part: SURVEY §8 f1, not built yet)")
        y_c = None if y is None else _dptr(_as_1d(y, "y", self.num_data))
        Xp = np.asfortranarray(np.asarray(gp_coords_pred, dtype=np.float64))
        npred = Xp.shape[0]
        cp_c = None if cov_pars is None else _dptr(_as_1d(cov_pars, "cov_pars", self.num_cov_pars))
        xp_c = None
        if X_pred is not None:  # covariates at the prediction points: X_pred beta is added to the mean (basic.py:6360-6380)
            X_pred = np.asarray(X_pred, dtype=np.float64)
            if X_pred.ndim == 1:
                X_pred = X_pred.reshape(-1, 1)
            if X_pred.shape[0] != npred:
                raise GPBoostError("Incorrect number of data points in X_pred")
            self._Xpred_c = np.ascontiguousarray(X_pred.flatten(order="F"))
            xp_c = _dptr(self._Xpred_c)
        cl_c = self._cluster_ids_pred_ptr(cluster_ids_pred, npred)
        self._safe_call(self._LIB.GPB_SetPredictionData(
            self.handle, ctypes.c_int32(npred), cl_c, None, None, _dptr(Xp), None, xp_c,
            c_str(vecchia_pred_type) if vecchia_pred_type else None, ctypes.c_int(num_neighbors_pred), ctypes.c_double(-1.),
            ctypes.c_int(-1), ctypes.c_int(-1)))
        out = np.zeros(npred * (2 if predict_var else 1), dtype=np.float64)
        self._safe_call(self._LIB.GPB_PredictREModel(
            self.handle, y_c, ctypes.c_int32(npred), _dptr(out), ctypes.c_bool(False), ctypes.c_bool(predict_var),
            ctypes.c_bool(predict_response), ctypes.c_bool(False), ctypes.c_bool(False), ctypes.c_int(0), ctypes.c_int(0),
            cl_c, None, None, _dptr(Xp), None, cp_c, xp_c, ctypes.c_bool(True), None, None))
        return {"mu": out[:npred].copy(), "var": out[npred:].copy() if predict_var else None}

    def _cluster_ids_pred_ptr(self, cluster_ids_pred, npred):
        """int32 labels of the independent realizations at the prediction points (basic.py: cluster_ids_pred); a label without training
        data predicts from the prior"""
        if cluster_ids_pred is None:
            return None
        self._cluster_ids_pred_c = np.ascontiguousarray(np.asarray(cluster_ids_pred).reshape(-1).astype(np.int32))
        if len(self._cluster_ids_pred_c) != npred:
            raise ValueError("Incorrect number of data points in 'cluster_ids_pred'")
        return self._cluster_ids_pred_c.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))

    def set_prediction_data(self, gp_coords_pred=None, vecchia_pred_type=None, num_neighbors_pred=None, X_pred=None,
                            cluster_ids_pred=None):
        """Set the prediction data (GPModel.set_prediction_data, basic.py): the GP coordinates of the validation data the GPBoost
        algorithm predicts at with `use_gp_model_for_validation=True`."""
        if gp_coords_pred is None and X_pred is None and vecchia_pred_type is None and num_neighbors_pred is None:
            raise ValueError("No prediction data given")
        coords_c, npred = None, 0
        if gp_coords_pred is not None:
            gp_coords_pred = np.asarray(gp_coords_pred, dtype=np.float64)
            if gp_coords_pred.ndim == 1:
                gp_coords_pred = gp_coords_pred.reshape(-1, 1)
            if gp_coords_pred.ndim != 2 or gp_coords_pred.shape[1] != self.dim_coords:
                raise ValueError("Incorrect number of dimensions / columns in 'gp_coords_pred'")
            npred = gp_coords_pred.shape[0]
            self._coords_pred_c = np.asfortranarray(gp_coords_pred)
            coords_c = _dptr(self._coords_pred_c)
        xp_c = None
        if X_pred is not None:
            X_pred = np.asarray(X_pred, dtype=np.float64)
            if X_pred.ndim == 1:
                X_pred = X_pred.reshape(-1, 1)
            if npred and X_pred.shape[0] != npred:
                raise ValueError("Incorrect number of data points in 'X_pred'")
            npred = X_pred.shape[0]
            self._Xpred_saved_c = np.ascontiguousarray(X_pred.flatten(order="F"))
            xp_c = _dptr(self._Xpred_saved_c)
        cl_c = self._cluster_ids_pred_ptr(cluster_ids_pred, npred) if cluster_ids_pred is not None and npred else None
        if cluster_ids_pred is not None and not npred:
            raise ValueError("'cluster_ids_pred' needs 'gp_coords_pred'")
        self._safe_call(self._LIB.GPB_SetPredictionData(
            self.handle, ctypes.c_int32(npred), cl_c, None, None, coords_c, None, xp_c,
            c_str(vecchia_pred_type) if vecchia_pred_type else None,
            ctypes.c_int(-1 if num_neighbors_pred is None else int(num_neighbors_pred)), ctypes.c_double(-1.),
            ctypes.c_int(-1), ctypes.c_int(-1)))
        if gp_coords_pred is not None:
            self.prediction_data_is_set = True
        return self

    prediction_data_is_set = False

    # ---- CUDA-build extensions ------------------------------------------------------------------------
    def response_gradient(self, y):
        """Psi^-1 y / sigma^2 at the current covariance parameters (what the boosting objective consumes)."""
        y = _as_1d(y, "y", self.num_data).copy()
        self._safe_call(self._LIB.GPB200_CalcGradient(self.handle, _dptr(y)))
        return y

    def device_engine(self):
        eng = ctypes.c_void_p()
        self._safe_call(self._LIB.GPB200_GetDeviceEngine(self.handle, ctypes.byref(eng)))
        return eng
