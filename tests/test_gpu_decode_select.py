"""GPU: the greedy choice of a decode step (`wts_decode_select`) and the filtered log-softmax rows
(`wts_filtered_logprobs`) against upstream's logit filters (SuppressBlank, SuppressTokens, ApplyTimestampRules) followed
by argmax / log_softmax, on crafted logit rows that reach every branch of the timestamp rules, in the three vocabulary
layouts (51864 `.en`, 51865 multilingual, 51866 large-v3)."""
import ctypes

import numpy as np
import pytest
import torch

from whisper_timestamped import model_zoo as zoo

import oracle_engine  # noqa: F401  (puts oracle/upstream on sys.path: `whisper` below is the oracle stand-in)

N_CTX, SAMPLE_LEN = 448, 224
SPACE = 220                                 # encode(" ") of the Whisper vocabularies: blank at the first sampled position


class TokStandIn:
    """The tokenizer attributes upstream's logit filters read."""

    def __init__(self, n_vocab):
        self.eot, self.sot, _, self.timestamp_begin = zoo.special_token_layout(n_vocab)
        self.no_timestamps = self.timestamp_begin - 1

    def encode(self, s):
        assert s == " "
        return [SPACE]


def suppress_list(tok):
    """A suppress set with text tokens, control tokens and one timestamp."""
    return sorted({1, 5, 221, 1000, 40000, tok.sot, tok.sot + 1, tok.no_timestamps - 1, tok.timestamp_begin + 7})


def upstream_filtered(logits, tokens, n_prompt, tok, suppress, max_initial_ts):
    """One row of logits (1-D tensor, float32 or float64) after upstream's greedy-decoding logit filters, in the order
    DecodingTask applies them.  tokens: the whole token row so far (prompt + sampled)."""
    from whisper.decoding import ApplyTimestampRules, SuppressBlank, SuppressTokens
    x = logits.clone()[None]
    t = torch.as_tensor(list(tokens), dtype=torch.long)[None]
    for f in (SuppressBlank(tok, n_prompt), SuppressTokens(suppress), ApplyTimestampRules(tok, n_prompt, max_initial_ts)):
        f.apply(x, t)
    return x[0]


def _cfg(nat, V, tok, mit):
    return nat.DecodeCfg(n_vocab=V, eot=tok.eot, timestamp_begin=tok.timestamp_begin, no_timestamps=tok.no_timestamps,
                         max_initial_ts=-1 if mit is None else mit, sample_len=SAMPLE_LEN, n_ctx=N_CTX, tokens_ld=N_CTX + 1)


def _cases(V, rng):
    """(name, tokens, n_prompt, logits float32 [V]) of one row each."""
    tok = TokStandIn(V)
    eot, tsb = tok.eot, tok.timestamp_begin
    sot_seq = [tok.sot, tok.sot + 1, tok.sot + 1 + 99 + 1]     # <|sot|> <|en|> <|transcribe|>-like prompt
    P = len(sot_seq)

    def base():
        x = rng.normal(0.0, 2.0, V).astype(np.float32)
        x[tsb:] += 1.0
        x[eot] = -5.0
        return x

    def text(n):
        return [int(t) for t in rng.integers(300, 30000, n)]

    out = []
    # first sampled position: text and eot forbidden (blank + the timestamp rule), max_initial_timestamp caps the first
    # timestamp; the largest timestamp sits past the cap
    x = base()
    x[tsb + 120] = 20.0
    x[tsb + 30] = 15.0
    x[SPACE] = 40.0
    out.append(("first", sot_seq, P, x))
    # last two sampled tokens timestamps: every timestamp forbidden
    x = base()
    x[tsb + 90] = 30.0
    out.append(("ts_ts", sot_seq + text(4) + [tsb + 10, tsb + 40, tsb + 40], P, x))
    # last a timestamp, penultimate text: text below eot forbidden, timestamps from the last one on (tl) allowed
    x = base()
    x[tsb + 40] = 25.0
    x[tsb + 39] = 30.0
    x[500] = 35.0
    out.append(("text_ts", sot_seq + [tsb + 2] + text(5) + [tsb + 40], P, x))
    # last text after a timestamp: the floor is tl + 1, tl itself forbidden
    x = base()
    x[tsb:] += 10.0
    x[tsb + 40] = 40.0
    x[tsb + 42] = 35.0
    out.append(("floor", sot_seq + [tsb + 2] + text(3) + [tsb + 40] + text(2), P, x))
    # no earlier timestamp: every timestamp allowed, the maximum at timestamp_begin itself
    x = base()
    x[tsb:] += 10.0
    x[tsb] = 30.0
    out.append(("no_ts_yet", sot_seq + text(6), P, x))
    # timestamp mass just above / just below the best text token (log-space margin 2e-3)
    for name, margin in (("mass_above", 2e-3), ("mass_below", -2e-3)):
        x = base()
        x[:tsb] = np.minimum(x[:tsb], 3.0)
        x[700] = 5.0
        x[tsb:] = -50.0
        k = 9
        x[tsb + 20:tsb + 20 + k] = np.float32(5.0 + margin - np.log(k))
        out.append((name, sot_seq + text(3), P, x))
    # bit-equal maxima in different warps of the 1024-thread CTA: the lowest index wins
    x = base()
    x[1005] = 30.0                          # thread 1005 (warp 31)
    x[2 * 1024 + 40] = 30.0                 # thread 40 (warp 1), higher index
    out.append(("tie_text_text", sot_seq + text(3), P, x))
    x = base()
    x[tsb:] = -50.0
    j = tsb + (1024 - tsb % 1024) + 3       # a timestamp on thread 3 (warp 0)
    x[1023] = 30.0                          # the text token on thread 1023 (warp 31)
    x[j] = 30.0
    out.append(("tie_text_ts", sot_seq + text(3), P, x))
    # eot chosen: done = 1, no token appended
    x = base()
    x[eot] = 40.0
    out.append(("eot", sot_seq + text(5), P, x))
    # the decoding limit via sample_len (n + 1 == sample_len) and via n_ctx (n_tokens + 1 > n_ctx)
    x = base()
    out.append(("limit_sample_len", sot_seq + text(SAMPLE_LEN - 1), P, x))
    x = base()
    long_prompt = [tok.sot - 1] + text(N_CTX - SAMPLE_LEN + 2 - 1 - P) + sot_seq
    out.append(("limit_n_ctx", long_prompt + text(N_CTX - len(long_prompt)), len(long_prompt), x))
    return tok, out


@pytest.mark.gpu
@pytest.mark.parametrize("V", [51864, 51865, 51866])
@pytest.mark.parametrize("mit", [50, None])
def test_decode_select_matches_upstream_filters(V, mit):
    from whisper_timestamped import _native as nat
    dev = "cuda"
    rng = np.random.default_rng(V + (mit or 0))
    tok, cases = _cases(V, rng)
    suppress = suppress_list(tok)
    blank = [SPACE, tok.eot]
    # one row per case, with finished rows in between (they must stay untouched)
    rows = []
    for c in cases:
        rows.append(c)
        if len(rows) % 3 == 2:
            rows.append(None)
    B = len(rows)
    ldl = V + 40
    logits = torch.full((B, ldl), 7.0, dtype=torch.float32)
    tokens = torch.zeros((B, N_CTX + 1), dtype=torch.int32)
    n_tokens = torch.ones(B, dtype=torch.int32)
    n_prompt = torch.ones(B, dtype=torch.int32)
    done = torch.zeros(B, dtype=torch.int32)
    for b, c in enumerate(rows):
        if c is None:
            done[b] = 1 + b % 2
            tokens[b, :3] = torch.tensor([tok.sot, 11, 12])
            n_tokens[b], n_prompt[b] = 3, 1
            continue
        _, t, npr, x = c
        tokens[b, :len(t)] = torch.tensor(t, dtype=torch.int32)
        n_tokens[b], n_prompt[b] = len(t), npr
        logits[b, :V] = torch.from_numpy(x)
    lp_ld = SAMPLE_LEN + 1
    host = dict(logits=logits, tokens=tokens, n_tokens=n_tokens, n_prompt=n_prompt, done=done)
    d = {k: v.to(dev) for k, v in host.items()}
    sup = torch.zeros(V, dtype=torch.uint8, device=dev)
    sup[torch.tensor(suppress, device=dev)] = 1
    blk = torch.zeros(V, dtype=torch.uint8, device=dev)
    blk[torch.tensor(blank, device=dev)] = 1
    logprobs = torch.full((B, lp_ld), 3.0, device=dev)
    full = torch.full((B, lp_ld, V), 5.0, device=dev)
    last_full = torch.full((B, V), 6.0, device=dev)
    rows_out = torch.full((B, V), 4.0, device=dev)
    cfg = _cfg(nat, V, tok, mit)
    st = nat.stream_ptr(dev)
    nat.check(nat.lib.wts_filtered_logprobs(d["logits"].data_ptr(), ldl, ctypes.byref(cfg), sup.data_ptr(), blk.data_ptr(),
                                            d["tokens"].data_ptr(), d["n_tokens"].data_ptr(), d["n_prompt"].data_ptr(),
                                            rows_out.data_ptr(), B, st), "wts_filtered_logprobs")
    torch.cuda.synchronize()
    for k, v in host.items():                                          # rows only: no state changes
        assert torch.equal(d[k].cpu(), v), k
    nat.check(nat.lib.wts_decode_select(d["logits"].data_ptr(), ldl, ctypes.byref(cfg), sup.data_ptr(), blk.data_ptr(),
                                        d["tokens"].data_ptr(), d["n_tokens"].data_ptr(), d["n_prompt"].data_ptr(),
                                        d["done"].data_ptr(), logprobs.data_ptr(), lp_ld, full.data_ptr(),
                                        last_full.data_ptr(), B, st), "wts_decode_select")
    torch.cuda.synchronize()
    g = {k: v.cpu() for k, v in d.items()}
    logprobs, full, last_full, rows_out = logprobs.cpu(), full.cpu(), last_full.cpu(), rows_out.cpu()
    seen = set()
    for b, c in enumerate(rows):
        if c is None:
            assert int(g["done"][b]) == int(done[b]) and torch.equal(g["tokens"][b], tokens[b])
            assert int(g["n_tokens"][b]) == int(n_tokens[b])
            assert bool((logprobs[b] == 3.0).all()) and bool((full[b] == 5.0).all()) and bool((last_full[b] == 6.0).all())
            continue
        name, t, npr, x = c
        n = len(t) - npr
        filt = upstream_filtered(torch.from_numpy(x), t, npr, tok, suppress, mit)
        ref_lp = torch.log_softmax(filt, -1)
        choice = int(filt.argmax())
        row = full[b, n]
        fin = torch.isfinite(ref_lp)
        assert torch.equal(torch.isfinite(row), fin), (name, torch.nonzero(torch.isfinite(row) != fin)[:5].flatten())
        err = float((row[fin] - ref_lp[fin]).abs().max())
        assert err <= 1e-5, (name, err)
        assert torch.equal(rows_out[b], row), name                     # the same row from wts_filtered_logprobs
        assert abs(float(logprobs[b, n]) - float(ref_lp[choice])) <= 1e-5, name
        assert float(logprobs[b, n]) == float(row[choice]), name
        limit = n + 1 >= SAMPLE_LEN or len(t) + 1 > N_CTX
        if choice == tok.eot:
            assert int(g["done"][b]) == 1 and int(g["n_tokens"][b]) == len(t), name
            assert torch.equal(g["tokens"][b], tokens[b]), name
        else:
            assert int(g["tokens"][b, len(t)]) == choice, (name, int(g["tokens"][b, len(t)]), choice)
            assert int(g["n_tokens"][b]) == len(t) + 1, name
            assert int(g["done"][b]) == (2 if limit else 0), name
            assert torch.equal(g["tokens"][b, :len(t)], tokens[b, :len(t)]), name
        if limit:
            assert torch.equal(last_full[b], row), name
        else:
            assert bool((last_full[b] == 6.0).all()), name
        seen.add((name, choice))
    # the crafted rows reach the branches they were made for
    ch = dict(seen)
    tsb, eot = tok.timestamp_begin, tok.eot
    assert ch["first"] == (tsb + 30 if mit is not None else tsb + 120)
    assert ch["ts_ts"] < tsb and ch["text_ts"] == tsb + 40 and ch["floor"] == tsb + 42
    assert ch["no_ts_yet"] == tsb and ch["mass_above"] == tsb + 20 and ch["mass_below"] == 700
    assert ch["tie_text_text"] == 1005 and ch["tie_text_ts"] == 1023 and ch["eot"] == eot
    assert ch["limit_sample_len"] != eot and ch["limit_n_ctx"] != eot
