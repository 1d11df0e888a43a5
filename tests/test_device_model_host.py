"""CPU tests of the resolver that turns a pipeline's ``model`` argument into the form the device path runs
(``pipelines._device_model``): a fit tuple, a compiled model or a host callable."""
import numpy as np
import pytest
from sklearn import ensemble

from pyimsegm_b200 import graph_cuts, pipelines as pl
from pyimsegm_b200.class_models import CompiledModel, compile_model


@pytest.fixture(scope='module')
def forest():
    rng = np.random.RandomState(0)
    x = rng.uniform(0, 1, (120, 3))
    return ensemble.RandomForestClassifier(n_estimators=4, max_depth=4, random_state=0).fit(x, (x[:, 0] > 0.5).astype(int))


def test_fit_tuple_and_compiled_model_pass_through(forest):
    fit = pl._fit_model(3, True)
    assert pl._device_model(fit, 3) is fit
    assert pl._device_model(fit, None) is fit
    cm = compile_model(forest)
    assert isinstance(cm, CompiledModel)
    assert pl._device_model(cm, 3) is cm
    assert pl._device_model(cm, None) is cm


def test_forest_of_matching_width_compiles(forest):
    cm = pl._device_model(forest, 3)
    assert isinstance(cm, CompiledModel) and cm.n_features_in == 3


def test_bound_predict_proba_is_unwrapped(forest):
    cm = pl._device_model(forest.predict_proba, 3)
    assert isinstance(cm, CompiledModel) and cm.digest == compile_model(forest).digest


@pytest.mark.parametrize('model', ['estimator', 'bound'])
def test_host_predict_proba_otherwise(forest, monkeypatch, model):
    m = forest if model == 'estimator' else forest.predict_proba
    assert pl._device_model(m, 4) == forest.predict_proba          # wrong width
    assert pl._device_model(m, None) == forest.predict_proba       # not a resident table
    monkeypatch.setattr(graph_cuts, 'USE_DEVICE_PREDICT', False)
    assert pl._device_model(m, 3) == forest.predict_proba


def test_plain_function_stays(forest):
    def proba_fn(features):
        return forest.predict_proba(features)

    assert pl._device_model(proba_fn, 3) is proba_fn
    assert pl._device_model(proba_fn, None) is proba_fn


def test_fit_model_takes_max_iter():
    assert pl._fit_model(3, True, max_iter=99) == ('fit', 3, True, 99)
    kind, n_init, n_iter = graph_cuts.class_model_spec('GMM', 3, 50)
    assert pl._fit_model(3, True, max_iter=50) == ('fit', 3, True, 50, kind, n_init, None)
    assert pl._fit_spec(pl._fit_model(3, True, max_iter=50)) == (3, True, 50, 'GMM', 7, None)
