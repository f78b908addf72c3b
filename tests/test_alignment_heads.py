"""`word_alignment_most_top_layers=k` and checkpoints without an alignment-head table: the product's host logic with the
CPU OracleEngine against the unmodified reference (tests/golden/heads/*.json, made by tests/golden/make_heads_golden.py).
The large-v3 cases take minutes per window through the fp32 CPU stand-in: they run here only with WTS_SLOW=1 (the GPU
suite runs them through the CUDA engine)."""
import contextlib
import glob
import io
import json
import os
from types import SimpleNamespace

import pytest

from whisper_timestamped import model_zoo as zoo
from whisper_timestamped.synthetic_audio import synthetic_speech
from whisper_timestamped.transcribe import top_layers_heads, transcribe_timestamped

from test_host_e2e import CaptureWarnings, compare, norm_warnings, stitch_cuts

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(glob.glob(os.path.join(HERE, "golden", "heads", "*.json")))


def case_heads(g):
    dims = zoo.DIMS[g["model"]]
    return zoo.ALIGNMENT_HEADS[g["model"]] if g["table_heads"] else zoo.default_alignment_heads(dims)


def heads_oracle_engine(model, heads):
    """The CPU OracleEngine plus the per-call head set transcribe() asks for (`set_alignment_heads`; None restores
    the heads it was built with)."""
    from oracle_engine import OracleEngine

    class HeadsOracleEngine(OracleEngine):
        def set_alignment_heads(self, heads=None):
            self.heads = list(self.model_heads if heads is None else heads)

    eng = HeadsOracleEngine(model, heads)
    eng.model_heads = list(heads)
    return eng


def run_oracle(g):
    from oracle_engine import build_oracle_model
    dims = zoo.DIMS[g["model"]]
    sd = zoo.synthetic_state_dict(dims, seed=g["model_seed"], **g["model_kwargs"])
    heads = case_heads(g)
    om = build_oracle_model(dims, sd, heads)
    eng = heads_oracle_engine(om, heads)
    shim = SimpleNamespace(dims=dims, is_multilingual=om.is_multilingual, num_languages=om.num_languages)
    kw = dict(g["transcribe_kwargs"])
    if "chunks" in g:
        kw["chunks"] = g["chunks"]
    with CaptureWarnings() as cap, contextlib.redirect_stdout(io.StringIO()):
        res = transcribe_timestamped(shim, synthetic_speech(*g["audio"]), engine=eng, **kw)
    return res, cap.messages


def check_golden(g, res, warns, conf_tol):
    if "chunks" in g:
        ref, ref_warns = stitch_cuts(g)
        compare(res, ref, conf_tol=conf_tol, time_tol=1e-6)
    else:
        ref, ref_warns = g["result"], g["warnings"]
        compare(res, ref, conf_tol=conf_tol)
    if warns is not None:
        assert norm_warnings(warns) == norm_warnings(ref_warns)


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-5] for p in CASES])
def test_host_logic_matches_heads_golden(path):
    g = json.load(open(path))
    if g["model"] != "tiny" and os.environ.get("WTS_SLOW") != "1":
        pytest.skip("large model: GPU test (WTS_SLOW=1 runs it through the CPU stand-in)")
    res, warns = run_oracle(g)
    check_golden(g, res, warns, conf_tol=1.5e-3)


def test_goldens_decode_like_the_table_goldens():
    """The head set changes no token: every heads/ golden has the segments and tokens of the table golden on the same
    audio seed (only word times and confidences may differ)."""
    by_audio = {}
    for p in glob.glob(os.path.join(HERE, "golden", "*.json")):
        g = json.load(open(p))
        if "audio" in g and g.get("model_kwargs") is not None:
            by_audio[(g["model"], tuple(g["audio"]), "chunks" in g)] = g
    assert CASES
    for p in CASES:
        g = json.load(open(p))
        base = by_audio[(g["model"], tuple(g["audio"]), "chunks" in g)]
        segs = [c["result"]["segments"] for c in g["cuts"]] if "chunks" in g else [g["result"]["segments"]]
        base_segs = [c["result"]["segments"] for c in base["cuts"]] if "chunks" in base else [base["result"]["segments"]]
        assert [[s["tokens"] for s in x] for x in segs] == [[s["tokens"] for s in x] for x in base_segs], p


def test_top_layers_heads_layer_major_and_clipped():
    assert top_layers_heads(4, 6, 2) == [(2, h) for h in range(6)] + [(3, h) for h in range(6)]
    assert top_layers_heads(4, 6, 9) == [(l, h) for l in range(4) for h in range(6)]
    assert len(top_layers_heads(32, 20, 6)) == 120
    assert top_layers_heads(32, 20, 16) == zoo.default_alignment_heads(zoo.DIMS["large-v3"])


@pytest.mark.parametrize("k", [0, -1])
def test_nonpositive_top_layers_asserts(k):
    with pytest.raises(AssertionError, match="strictly positive"):
        transcribe_timestamped(SimpleNamespace(), None, word_alignment_most_top_layers=k)
