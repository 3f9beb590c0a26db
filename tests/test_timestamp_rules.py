"""Whisper's timestamp rules on the CPU: the oracle's restatement against transformers' WhisperTimeStampLogitsProcessor
(golden tests/golden/timestamp_rules_hf.npz), the golden's coverage of every rule, the transcripts of the
timestamp-scripted test model, and the host-side plumbing of timestamp mode."""
import functools
import os

import numpy as np
import pytest
import torch

from oracle.whisper_ref import WhisperOracle
from tests.ts_oracle import RULES, TimestampOracle, apply_timestamp_rules, check_invariants
from willow_inference_server_b200 import audio, models, weights as W

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "timestamp_rules_hf.npz")
TS_PROMPT = [50258, 50259, 50359]            # sot, <|en|>, transcribe: no <|notimestamps|>
SCRIPT, RAMP, TS_SCRIPT = (4, 3.3, 1.67), (8, 12.0), (2, 5, 8)


def golden_rows():
    g = np.load(GOLDEN)
    for i in range(g["geom"].shape[0]):
        V, eot, no_ts = (int(v) for v in g["geometries"][g["geom"][i]])
        gen = int(g["gen"][i])
        x = np.random.default_rng(int(g["seed"][i])).standard_normal(V, dtype=np.float32) * np.float32(3.0)
        x[no_ts + 1:] += g["shift"][i]
        dis = np.unpackbits(g["disabled"][i])[:V].astype(bool)
        yield dict(V=V, eot=eot, no_ts=no_ts, gen=gen, hist=[int(t) for t in g["hist"][i][:gen]],
                   max_init=int(g["max_init"][i]), logits=x, disabled=dis)


def oracle_disabled(row, disable=()):
    out = apply_timestamp_rules(torch.from_numpy(row["logits"][None].copy()), [row["hist"]], row["gen"],
                                no_timestamps=row["no_ts"], eot=row["eot"], max_initial_timestamp_index=row["max_init"],
                                disable=disable)[0].numpy()
    return np.isneginf(out)


def test_oracle_rules_match_hf_golden():
    rows = list(golden_rows())
    assert len(rows) >= 60 and {r["V"] for r in rows} == {51864, 51865, 51866}
    for i, row in enumerate(rows):
        got = oracle_disabled(row)
        assert np.array_equal(got, row["disabled"]), (i, row["V"], row["gen"], row["hist"], np.flatnonzero(got != row["disabled"])[:8])


@pytest.mark.parametrize("rule", RULES)
def test_golden_covers_every_rule(rule):
    # with any one rule missing from the oracle, some golden row disagrees: the golden reaches every branch
    assert any(not np.array_equal(oracle_disabled(row, (rule,)), row["disabled"]) for row in golden_rows())


@functools.lru_cache(maxsize=1)
def ts_oracle():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=2, n_dec_layers=2)
    tensors = W.synth_engine_tensors(dims, seed=11, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    buf = np.zeros(W.blob_nbytes(tensors), np.uint8)
    W.write_blob_into(buf, dims, tensors)
    o = TimestampOracle.from_blob(buf)
    ts_oracle.plain = WhisperOracle.from_blob(buf)
    from oracle import logmel as om

    durations = [61440, 160000, 480000, 171008, 30000, 467968]
    mel = om.log_mel_batch([om.synth_utterance(m, 100 + i) for i, m in enumerate(durations)])
    return dims, o, mel, o.encode(mel)


@pytest.mark.parametrize("beam", [1, 3])
def test_oracle_timestamp_transcripts_satisfy_the_invariants(beam):
    dims, o, mel, enc = ts_oracle()
    n = 6 if beam == 1 else 3
    res = o.generate(mel[:n], [TS_PROMPT] * n, beam_size=beam, enc=enc[:n])
    segs = [check_invariants(r.sequences_ids[0], dims) for r in res]
    assert min(segs) >= 2, segs
    assert len({tuple(r.sequences_ids[0]) for r in res}) >= 2  # the transcripts depend on the audio
    for mi in (0, 5):
        for r in o.generate(mel[:n], [TS_PROMPT] * n, beam_size=beam, enc=enc[:n], max_initial_timestamp_index=mi):
            check_invariants(r.sequences_ids[0], dims, mi)


@pytest.mark.parametrize("rule", RULES + ("clamp",))
def test_every_rule_changes_a_transcript(rule):
    dims, o, mel, enc = ts_oracle()
    base = o.generate(mel, [TS_PROMPT] * 6, beam_size=1, enc=enc)
    if rule == "clamp":
        alt = o.generate(mel, [TS_PROMPT] * 6, beam_size=1, enc=enc, max_initial_timestamp_index=1000)
    else:
        alt = o.generate(mel, [TS_PROMPT] * 6, beam_size=1, enc=enc, disable=(rule,))
    assert any(a.sequences_ids != b.sequences_ids for a, b in zip(alt, base))


def test_notimestamps_prompt_is_untouched_by_the_subclass():
    dims, o, mel, enc = ts_oracle()
    prompt = TS_PROMPT + [dims.no_timestamps]
    for beam in (1, 2):
        a = o.generate(mel[:2], [prompt] * 2, beam_size=beam, enc=enc[:2])
        b = ts_oracle.plain.generate(mel[:2], [prompt] * 2, beam_size=beam, enc=enc[:2])
        assert [r.sequences_ids for r in a] == [r.sequences_ids for r in b]


def test_ts_script_changes_only_the_decoder_positions():
    dims = W.WhisperDims(d_model=128, n_heads=2, n_enc_layers=1, n_dec_layers=1)
    a = W.synth_state_dict(dims, seed=3, eot_ramp=RAMP, script=SCRIPT)
    b = W.synth_state_dict(dims, seed=3, eot_ramp=RAMP, script=SCRIPT, ts_script=None)
    c = W.synth_state_dict(dims, seed=3, eot_ramp=RAMP, script=SCRIPT, ts_script=TS_SCRIPT)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    assert [k for k in a if not np.array_equal(a[k], c[k])] == ["model.decoder.embed_positions.weight"]
    with pytest.raises(ValueError):
        W.synth_state_dict(dims, seed=3, ts_script=TS_SCRIPT)


class _FakeHandle:
    def __init__(self):
        self.calls = []

    def set_option(self, k, v):
        pass

    def dims(self):
        return {"n_vocab": 51865, "n_langs": 99, "no_timestamps": 50363, "lang_first": 50259}

    def generate(self, mel, prompts, *args, **kw):
        self.calls.append(kw)
        return [[] for _ in range(mel.shape[0])], [0.0] * mel.shape[0]


def test_generate_selects_timestamp_mode_from_the_prompt():
    h = _FakeHandle()
    m = models.Whisper(None, device="cuda", _handles=[h])
    mel = np.zeros((2, 80, 3000), np.float32)
    m.generate(mel, [TS_PROMPT] * 2)
    m.generate(mel, [TS_PROMPT + [50363]] * 2, max_initial_timestamp_index=7)
    m.generate(mel, [TS_PROMPT] * 2, max_initial_timestamp_index=0)
    assert [(c["timestamps"], c["max_initial_timestamp_index"]) for c in h.calls] == [(True, 50), (False, 7), (True, 0)]
    with pytest.raises(ValueError):
        m.generate(mel, [TS_PROMPT, TS_PROMPT + [50363]])  # one call decodes in one mode
    with pytest.raises(ValueError):
        m.generate(mel, [TS_PROMPT] * 2, max_initial_timestamp_index=-1)
    with pytest.raises(ValueError):
        m.generate(mel, [TS_PROMPT] * 2, max_initial_timestamp_index=1.5)


def test_transcribe_long_rejects_timestamps_over_several_windows(monkeypatch):
    class Tok:
        all_special_ids = [50257, 50258]

    class Engine:
        dims = {"no_timestamps": 50363}

        def generate(self, features, prompts, **kw):
            return [models.WhisperGenerationResult([[1, 2]]) for _ in range(features.array.shape[0])]

    monkeypatch.setattr(audio, "log_mel_chunks", lambda a, handle=None: (np.zeros((2, 80, 3000), np.float32),
                                                                        [(352000, 0, 64000), (100000, 64000, 0)]))
    monkeypatch.setattr(audio, "log_mel_window", lambda a, handle=None: np.zeros((1, 80, 3000), np.float32))
    with pytest.raises(ValueError, match="timestamp"):
        audio.transcribe_long(Engine(), np.zeros(800000, np.float32), TS_PROMPT, Tok())
    assert audio.transcribe_long(Engine(), np.zeros(800000, np.float32), TS_PROMPT + [50363], Tok()).size >= 0
    assert audio.transcribe_long(Engine(), np.zeros(400000, np.float32), TS_PROMPT, Tok()).tolist() == [1, 2]
