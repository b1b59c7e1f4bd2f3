"""SFSORT's configuration contract without a GPU: constructor clamps and YAML defaults against the reference
(tests/golden/sfsort_contract.json), create_tracker("sfsort") resolution, the out-of-scope cases, and
BoxMOTSFSORTConfig against the reference's own ctypes binding."""
import ctypes
import json
import re
from pathlib import Path

import pytest

from boxmot_b200 import _lib
from boxmot_b200.trackers import SFSORT, SFSORT_YAML_DEFAULTS, TRACKER_DEFAULTS, resolve_tracker_args, sfsort_resolve

ROOT = Path(__file__).resolve().parents[1]
CONTRACT = json.loads((ROOT / "tests" / "golden" / "sfsort_contract.json").read_text())


@pytest.mark.parametrize("k", range(len(CONTRACT["resolved"])))
def test_constructor_clamps_match_reference(k):
    case = CONTRACT["resolved"][k]
    r = sfsort_resolve(**case["args"])
    for name, want in case["resolved"].items():
        if name in r:
            assert r[name] == want, name


def test_yaml_defaults_match_reference():
    assert SFSORT_YAML_DEFAULTS == CONTRACT["yaml"]
    assert "sfsort" not in TRACKER_DEFAULTS


def test_create_tracker_resolution():
    kind, cls, args = resolve_tracker_args("sfsort", overrides=dict(central_timeout=7, per_class=False, unknown=1))
    assert kind == "sfsort" and cls is SFSORT
    assert args == dict(SFSORT_YAML_DEFAULTS, central_timeout=7)


@pytest.mark.parametrize("kw", [dict(per_class=True), dict(is_obb=True)])
def test_out_of_scope_raises(kw):
    with pytest.raises(NotImplementedError):
        SFSORT(**kw)


def test_sfsort_config_layout_matches_reference_binding():
    fields = [[n, {_lib.c_float: "float", _lib.c_int: "int"}[t]] for n, t in _lib.BoxMOTSFSORTConfig._fields_]
    assert fields == CONTRACT["BoxMOTSFSORTConfig"]
    assert ctypes.sizeof(_lib.BoxMOTSFSORTConfig) == CONTRACT["sizeof_BoxMOTSFSORTConfig"]
    text = (ROOT / "include" / "boxmot_b200.h").read_text()
    body = re.search(r"typedef struct BoxMOTSFSORTConfig \{(.*?)\} BoxMOTSFSORTConfig;", text, flags=re.S).group(1)
    assert [d.split() for d in body.replace("\n", " ").split(";") if d.strip()] == [[t, n] for n, t in fields]
    assert _lib.TRACKER_SFSORT == 6 and "#define BOXMOT_B200_TRACKER_SFSORT 6" in text
