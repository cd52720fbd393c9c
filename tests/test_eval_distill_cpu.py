"""Host side of the distillation student's evaluation pass without a GPU: which policy `EvalStepsB200` runs for each training driver
(`driver_kind`), the refusal of other drivers, and `DistillStepsB200.evaluate`'s contract with the pass."""
from types import SimpleNamespace as NS

import pytest

from pulse_b200 import _lib
from pulse_b200.distill import DistillStepsB200
from pulse_b200.evaluation import EvalStepsB200, driver_kind
from pulse_b200.imz_rollout import ImZStepsB200
from pulse_b200.rollout import PlayStepsB200


class _Distill(DistillStepsB200):
    """A subclass of the driver: still the student's pass."""


@pytest.mark.parametrize("cls,kind", [(PlayStepsB200, "im"), (ImZStepsB200, "vr"), (DistillStepsB200, "distill"), (_Distill, "distill")])
def test_driver_kind(cls, kind):
    assert driver_kind(object.__new__(cls)) == kind


@pytest.mark.parametrize("driver", [NS(policy=None), NS(vae=None, sim={}), object()])
def test_other_drivers_are_refused_by_name(driver):
    for fn in (driver_kind, EvalStepsB200):
        with pytest.raises(_lib.PulseError) as e:
            fn(driver)
        msg = str(e.value)
        assert "PlayStepsB200 and ImZStepsB200" in msg and "DistillStepsB200" in msg and type(driver).__name__ in msg


def test_evaluate_holds_the_pass_and_returns_its_result(monkeypatch):
    """`evaluate` builds the pass over the driver with the hook and the pass options, keeps it as `eval_steps` and returns `run`'s
    result with the PMCP flags passed through."""
    from pulse_b200 import evaluation
    seen = {}

    class Pass:
        def __init__(self, driver, physics=None, **kw):
            seen.update(driver=driver, physics=physics, kw=kw)

        def run(self, dataset, auto_pmcp=False, auto_pmcp_soft=False):
            seen.update(dataset=dataset, pmcp=(auto_pmcp, auto_pmcp_soft), held=drv.eval_steps is self)
            return {"eval_info": {}}

    monkeypatch.setattr(evaluation, "EvalStepsB200", Pass)
    drv = object.__new__(DistillStepsB200)
    hook, ds = (lambda t: None), object()
    out = drv.evaluate(ds, physics=hook, auto_pmcp_soft=True, poll_every=4, use_graphs=False)
    assert out == {"eval_info": {}} and seen["held"] and seen["driver"] is drv and seen["physics"] is hook and seen["dataset"] is ds
    assert seen["pmcp"] == (False, True) and seen["kw"] == {"poll_every": 4, "use_graphs": False}
