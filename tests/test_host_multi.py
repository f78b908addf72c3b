"""transcribe(model, [audio, ...]) on the CPU host path (OracleEngine stand-ins): ONE call over several recordings must give,
per recording, what the unmodified reference gives on that recording alone (tests/golden/multi/*.json, produced by
tests/golden/make_multi_golden.py, and the groups of e2e goldens that share their options), with the same warnings and
the same stdout, one recording after the other."""
import contextlib
import glob
import io
import json
import os
from collections import defaultdict
from types import SimpleNamespace

import pytest

from test_host_e2e import CASES, CaptureWarnings, _is_big, compare, norm_warnings
from whisper_timestamped import model_zoo as zoo
from whisper_timestamped.synthetic_audio import synthetic_speech
from whisper_timestamped.transcribe import transcribe_timestamped

HERE = os.path.dirname(os.path.abspath(__file__))
MULTI = sorted(glob.glob(os.path.join(HERE, "golden", "multi", "*.json")))


def oracle_setup(model, model_seed, model_kwargs):
    from oracle_engine import OracleEngine, build_oracle_model
    dims = zoo.DIMS[model]
    sd = zoo.synthetic_state_dict(dims, seed=model_seed, **model_kwargs)
    heads = zoo.ALIGNMENT_HEADS[model]
    om = build_oracle_model(dims, sd, heads)
    shim = SimpleNamespace(dims=dims, is_multilingual=om.is_multilingual, num_languages=om.num_languages)
    return shim, OracleEngine(om, heads)


def run_files(model, eng, audios, **kw):
    out = io.StringIO()
    with CaptureWarnings() as cap, contextlib.redirect_stdout(out):
        res = transcribe_timestamped(model, audios, engine=eng, **kw)
    return res, cap.messages, out.getvalue()


def e2e_groups():
    """Existing e2e goldens that share model, model kwargs and transcribe kwargs: each group is one list call."""
    groups = defaultdict(list)
    for path in CASES:
        g = json.load(open(path))
        if "chunks" in g:
            continue
        key = json.dumps([g["model"], g["model_seed"], g["model_kwargs"], g["transcribe_kwargs"]], sort_keys=True)
        groups[key].append(path)
    return [sorted(p) for p in groups.values() if len(p) > 1]


GROUPS = e2e_groups()


@pytest.mark.parametrize("path", MULTI, ids=[os.path.basename(p)[:-5] for p in MULTI])
def test_one_call_over_files_matches_reference_per_file(path):
    if _is_big(path):
        pytest.skip("large model: GPU test (WTS_SLOW=1 runs it through the CPU stand-in)")
    g = json.load(open(path))
    model, eng = oracle_setup(g["model"], g["model_seed"], g["model_kwargs"])
    res, warns, stdout = run_files(model, eng, [synthetic_speech(*a) for a in g["audios"]], **g["transcribe_kwargs"])
    assert isinstance(res, list) and len(res) == len(g["files"])
    for r, item in zip(res, g["files"]):
        if "min_top2_gap" in item:
            assert item["min_top2_gap"]["gap"] >= 1e-4, item["min_top2_gap"]
        compare(r, item["result"])
    assert norm_warnings(warns) == norm_warnings([m for item in g["files"] for m in item["warnings"]])
    if "stdout" in g["files"][0]:
        assert stdout == "".join(item["stdout"] for item in g["files"])


@pytest.mark.parametrize("paths", GROUPS, ids=["+".join(os.path.basename(p)[4:-5] for p in ps) for ps in GROUPS])
def test_e2e_goldens_with_shared_options_in_one_call(paths):
    gs = [json.load(open(p)) for p in paths]
    if any(_is_big(p) for p in paths):
        pytest.skip("large model: GPU test (WTS_SLOW=1 runs it through the CPU stand-in)")
    model, eng = oracle_setup(gs[0]["model"], gs[0]["model_seed"], gs[0]["model_kwargs"])
    res, warns, stdout = run_files(model, eng, [synthetic_speech(*g["audio"]) for g in gs], **gs[0]["transcribe_kwargs"])
    for r, g in zip(res, gs):
        compare(r, g["result"])
    if all("warnings" in g for g in gs):
        assert norm_warnings(warns) == norm_warnings([m for g in gs for m in g["warnings"]])
    if all("stdout" in g for g in gs):
        assert stdout == "".join(g["stdout"] for g in gs)


def test_e2e_groups_are_the_expected_ones():
    names = sorted(tuple(os.path.basename(p)[4:-5] for p in ps) for ps in GROUPS)
    assert ("tiny_75s_cond", "tiny_short") in names
    assert ("tiny_detect_lang", "tiny_detect_lang_short") in names


def test_one_element_list_equals_scalar_call():
    g = json.load(open(os.path.join(HERE, "golden", "e2e_tiny_short.json")))
    model, eng = oracle_setup(g["model"], g["model_seed"], g["model_kwargs"])
    audio = synthetic_speech(*g["audio"])
    one, w1, o1 = run_files(model, eng, audio, **g["transcribe_kwargs"])
    many, w2, o2 = run_files(model, eng, (audio,), **g["transcribe_kwargs"])
    assert many == [one] and w1 == w2 and o1 == o2
    assert run_files(model, eng, [], **g["transcribe_kwargs"])[0] == []


def test_chunks_with_a_list_is_refused():
    with pytest.raises(NotImplementedError):
        transcribe_timestamped(SimpleNamespace(), [synthetic_speech(1.0, 1)], chunks=30.0, engine=object())
