import io
import os
import random
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.realpath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100, sm_90a; run with -m gpu)')


def random_dna(rnd, n, alphabet='ACGT'):
    return ''.join(rnd.choice(alphabet) for _ in range(n))


def mutate(rnd, s, rate):
    out = []
    for c in s:
        x = rnd.random()
        if x < rate / 3:
            continue
        if x < 2 * rate / 3:
            out.append(rnd.choice('ACGT'))
        elif x < rate:
            out.append(c)
            out.append(rnd.choice('ACGT'))
        else:
            out.append(c)
    return ''.join(out) or 'A'


@pytest.fixture(scope='session')
def sink():
    return io.StringIO()


_MODEL_CACHE = {}


def load_models(error_name, qscore_name):
    from badread_b200.error_model import ErrorModel
    from badread_b200.qscore_model import QScoreModel
    key = (error_name, qscore_name)
    if key not in _MODEL_CACHE:
        out = io.StringIO()
        _MODEL_CACHE[key] = (ErrorModel(error_name, out), QScoreModel(qscore_name, out))
    return _MODEL_CACHE[key]


@pytest.fixture(scope='session')
def engine():
    from badread_b200.engine import Engine
    eng = Engine(device=0, seed=1234)
    yield eng
    eng.close()
