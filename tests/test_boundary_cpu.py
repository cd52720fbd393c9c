"""CPU checks of the drop-in layer's CONTRACT: (1) every reference attribute / method name the stand-ins carry (tests/standins.CONTRACT)
occurs in the unmodified reference file it is cited from -- against the pairs recorded from those files (tests/golden/contract_names.json,
make_golden_contract.py); (2) every attribute the mixins read from `self` is either defined by the mixin, listed in the contract, or
private to the mixin (`_pulse*`) -- so the stand-ins cannot silently drift from what the mixins need."""
import ast
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_contract_names_exist_in_the_reference_sources():
    from tests.standins import CONTRACT
    with open(os.path.join(ROOT, "tests", "golden", "contract_names.json")) as f:
        recorded = {rel: set(names) for rel, names in json.load(f).items()}
    missing = [(rel, n) for side in CONTRACT.values() for rel, names in side.items() for n in names if n not in recorded.get(rel, ())]
    assert not missing, missing


def _self_attrs(path, class_name):
    tree = ast.parse(open(path).read())
    cls = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == class_name)
    reads, defined = set(), {n.name for n in cls.body if isinstance(n, ast.FunctionDef)}
    for node in ast.walk(cls):
        if isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name) and node.value.id == "self":
            reads.add(node.attr)
        if isinstance(node, ast.Call) and isinstance(node.func, ast.Name) and node.func.id == "getattr" and len(node.args) >= 2 \
                and isinstance(node.args[0], ast.Name) and node.args[0].id == "self" and isinstance(node.args[1], ast.Constant):
            reads.add(node.args[1].value)
    return reads, defined


@pytest.mark.parametrize("path,cls,side", [("pulse_b200/humanoid_im.py", "HumanoidImB200Mixin", "task"),
                                           ("pulse_b200/agent_mixins.py", "AMPAgentB200Mixin", "agent")])
def test_mixins_only_touch_contract_names(path, cls, side):
    from tests.standins import CONTRACT
    reads, defined = _self_attrs(os.path.join(ROOT, path), cls)
    allowed = set(n for names in CONTRACT[side].values() for n in names) | defined
    extra = {"device", "num_envs", "dt", "vec_env", "model", "optimizer", "obs_shape", "actions_num", "add_obs_noise", "_pulse"}   # generic BaseTask / A2CBase fields
    unknown = sorted(a for a in reads if a not in allowed and a not in extra and not a.startswith("_pulse"))
    assert not unknown, f"{cls} reads attributes that are not in tests/standins.CONTRACT: {unknown}"
