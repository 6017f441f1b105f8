import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (select with `-m gpu`)")


@pytest.fixture(params=["f64", "f32"])
def lin_reg_dtype(request, monkeypatch):
    """Mirror of the reference fixture (tests/test_linear_exprs.py:1184-1188): run under both plugin variants."""
    import polars_ds_extension_b200.config as cfg

    monkeypatch.setattr(cfg, "LIN_REG_EXPR_F64", request.param == "f64")
    return request.param
