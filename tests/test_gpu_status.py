"""GPU: what gpb200_last_error reports on an in-process group of virtual ranks (LocalGroupEngine).  Every collective call
clears the message of every rank before it runs, so a message left afterwards belongs to that call; the failures the
leader reports keep their text."""
import numpy as np
import pytest

from conftest import make_data

pytestmark = pytest.mark.gpu


def _errors(eng):
    return [e._lib.gpb200_last_error(e._h).decode() for e in eng.engines]


def test_collective_call_clears_every_rank():
    import gpb200
    X, y, _ = make_data(600, 2, 61)
    eng = gpb200.LocalGroupEngine(2, rb=1)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), gpb200.SEIso(0.1, 0.1), -0.5, engine=eng)
    with pytest.raises(ValueError, match="nb must be"):
        eng.engines[1].set_option("nb", 3)                  # rejected on rank 1 alone
    assert "nb must be" in _errors(eng)[1]
    eng.factorize(gp._theta_full(), -0.5)
    assert _errors(eng) == ["", ""]
    eng.solve(np.ones(eng.N))
    assert _errors(eng) == ["", ""]
    eng.close()


def test_leader_reports_group_failures():
    """a duplicate point under the noise kernel at negligible noise gives an exactly zero pivot"""
    import gpb200
    X, y, _ = make_data(400, 2, 47)
    X[350] = X[100]
    eng = gpb200.LocalGroupEngine(3, rb=1)
    gp = gpb200.GPE(X.T, y, gpb200.MeanZero(), gpb200.Noise(0.0), -0.5, engine=eng)
    with pytest.raises(ValueError, match="leader"):
        eng.engines[1].factorize(gp._theta_full(), -0.5)    # collective entry points go through the leader
    assert "leader" in _errors(eng)[1]
    with pytest.raises(gpb200.PosDefException):
        eng.factorize(gp._theta_full(), -40.0)
    errs = _errors(eng)
    assert errs[0].startswith("matrix is not positive definite; leading minor "), errs[0]
    assert errs[1:] == ["", ""]
    with pytest.raises(ValueError, match="factorize first"):
        eng.solve(np.ones(eng.N))                           # the failed factorisation left no factor on the leader
    eng.close()
