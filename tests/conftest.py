import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


@pytest.fixture(scope="session")
def tpch_tiny():
    """dbgen SF0.001 tables -- the data set the reference's golden snapshots were produced from"""
    from datagen import tpch
    return tpch.tables(0.001)


@pytest.fixture(scope="session")
def golden():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "tpch_sf0001_result.json")) as f:
        return json.load(f)["queries"]
