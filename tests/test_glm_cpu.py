"""GLM without a GPU: the IRLS oracle (tests/glm_oracle.py) against independent solvers on the data of the reference's
test_glm_family, the reference's convergence-failure case, the NaN stopping rule, and the host-side surface of
`linear_models.GLM` (constructor errors, unfitted state, repr, the loud failure without a CUDA device).

The reference checks GLM against statsmodels, which is not installed here; scikit-learn and SciPy stand in for it.
Its test_glm uses the scotland dataset that ships with statsmodels, so that case cannot be lifted."""
import numpy as np
import pytest

from tests.glm_oracle import LIFTED_FAMILIES, LIFTED_ITERS, faer_irls, lifted_case


def independent_fit(family: str, X: np.ndarray, y: np.ndarray):
    """(coefficients, bias) of the unpenalised maximum-likelihood fit, by a solver that shares no code with IRLS."""
    if family == "gaussian":
        from sklearn.linear_model import LinearRegression

        m = LinearRegression().fit(X, y)
        return m.coef_, float(m.intercept_)
    if family == "binomial":
        from sklearn.linear_model import LogisticRegression

        m = LogisticRegression(C=np.inf, solver="newton-cholesky", tol=1e-12, max_iter=1000).fit(X, y)
        return m.coef_.ravel(), float(m.intercept_[0])
    if family == "poisson":
        from sklearn.linear_model import PoissonRegressor

        m = PoissonRegressor(alpha=0.0, solver="newton-cholesky", tol=1e-12, max_iter=1000).fit(X, y)
        return m.coef_, float(m.intercept_)
    # gamma, inverse link (sklearn has no such model): BFGS on sum(y eta - ln eta), eta = X1 beta > 0, gradient
    # X1'(y - 1 / eta).  BFGS may report a precision loss near the optimum; the tolerance below is what is checked.
    from scipy.optimize import minimize

    X1 = np.column_stack([X, np.ones(len(y))])

    def fun(b):
        eta = X1 @ b
        return np.inf if np.any(eta <= 0.0) else float(np.sum(y * eta - np.log(eta)))

    b0 = np.zeros(X1.shape[1])
    b0[-1] = 1.0 / y.mean()
    r = minimize(fun, b0, jac=lambda b: X1.T @ (y - 1.0 / (X1 @ b)), method="BFGS", options={"gtol": 1e-12})
    return r.x[:-1], float(r.x[-1])


@pytest.mark.parametrize("family", LIFTED_FAMILIES)
def test_oracle_against_independent_solvers(family):
    X, y = lifted_case(family)
    beta, n_iter = faer_irls(np.column_stack([X, np.ones(len(y))]), y, family, 1e-8, 200)
    coef, bias = independent_fit(family, X, y)
    np.testing.assert_allclose(beta[:-1], coef, rtol=0, atol=1e-8)
    assert abs(beta[-1] - bias) < 1e-8
    assert n_iter == LIFTED_ITERS[family]


def test_oracle_convergence_failure_case():
    """The reference's test_glm_convergence_failure: poisson, no bias, max_iter=1, tol=1e-12 -> finite coefficients."""
    rng = np.random.RandomState(0)
    n, p = 200, 5
    X = rng.randn(n, p)
    y = np.exp(np.clip(X @ np.ones(p) * 0.2, -2, 2)) + rng.exponential(0.5, n)
    beta, n_iter = faer_irls(X, y, "poisson", 1e-12, 1)
    assert n_iter == 1 and np.all(np.isfinite(beta))


def test_oracle_nan_stops_the_loop():
    """log of a negative start gives NaN moments; f64::max ignores the NaN difference, so the loop ends after one
    iteration and returns NaN coefficients."""
    rng = np.random.RandomState(1)
    X = rng.randn(100, 3)
    beta, n_iter = faer_irls(X, -1.0 - rng.random(100), "poisson", 1e-8, 100)
    assert n_iter == 1 and np.all(np.isnan(beta))


def test_constructor_errors_and_defaults():
    from polars_ds_extension_b200.linear_models import GLM

    with pytest.raises(NotImplementedError):
        GLM(solver="lbfgs")
    with pytest.raises(ValueError, match="`max_iter` must be > 1."):
        GLM(max_iter=0)
    for bad in ("Poisson", "tweedie", "inverse_gaussian", ""):
        with pytest.raises(NotImplementedError):
            GLM(family=bad)
    g = GLM(tol=-1e-6, feature_names_in_=["a"])
    assert g._tol == 1e-6 and g._max_iter == 100 and not g._add_bias and g.feature_names_in_ == ["a"]
    assert GLM.__init__.__defaults__ == (False, "irls", "normal", 100, 1e-8, None)


def test_repr_and_unfitted_state():
    from polars_ds_extension_b200.linear_models import GLM

    names = {"gaussian": ("Identity", "Gaussian"), "normal": ("Identity", "Gaussian"), "poisson": ("Log", "Poisson"),
             "binomial": ("Logit", "Binomial"), "logistic": ("Logit", "Binomial"), "gamma": ("Inverse", "Gamma")}
    for fam, (link, var) in names.items():
        assert repr(GLM(family=fam)) == f"GLM:\nLink: {link}\nVariance: {var}"
    g = GLM(add_bias=True)
    assert not g.is_fit() and g.bias() == 0.0
    with pytest.raises(ValueError, match="Matrix is not learned yet."):
        g.coeffs()
    with pytest.raises(ValueError, match="Matrix is not learned yet."):
        g.predict(np.zeros((2, 2)))
    assert g.set_input_features(["x", "y"]) is g and g.feature_names_in_ == ["x", "y"]
    # the reference comments both out: GLM has neither
    assert not hasattr(GLM, "predict_df") and not hasattr(GLM, "from_values")


def test_glm_is_exported():
    import polars_ds_extension_b200.linear_models as lm

    assert "GLM" in lm.__all__ and lm.GLM.__name__ == "GLM"


def test_fit_fails_loudly_without_gpu():
    import torch

    from polars_ds_extension_b200.linear_models import GLM

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    X, y = lifted_case("poisson")
    with pytest.raises(ValueError, match="no usable CUDA device"):
        GLM(family="poisson").fit(X, y)
