"""Chunked streaming of the causal time-domain models (fcb_stream_*, B200Encodec.encode_stream / decode_stream) against the
whole clip through fcb_encode + fcb_decode_*: codes, quantized embeddings and waveform must be the same bits for every chunk
schedule, every batch size and both conv paths."""
import ctypes

import numpy as np
import pytest
import torch

from funcodec_b200 import _capi, get_config, init_state_dict
from oracle import encodec_oracle as O
from parity_utils import assert_codes_parity

pytestmark = pytest.mark.gpu

CAUSAL = ["soundstream_causal_small", "causal_lstm_small", "soundstream_16k_n32_ds320"]
_MODELS = {}


def _model(name, use_tc=1, seed=5, **kw):
    from funcodec_b200.encodec import B200Encodec
    key = (name, use_tc, seed, tuple(sorted(kw.items())))
    if key not in _MODELS:
        cfg = get_config(name)
        sd = init_state_dict(cfg, seed)
        _MODELS[key] = (cfg, sd, B200Encodec(cfg, sd, "cuda:0", options={"use_tc": use_tc}, **kw))
    return _MODELS[key]


def _wav(B, L, seed=11):
    g = torch.Generator().manual_seed(seed)
    return (0.1 * torch.randn(B, L, generator=g)).cuda()


def _schedule(kind, F, fmin):
    if kind == "single":
        return [F]
    out, pat = [fmin], ([1] if kind == "ones" else [3, 1, 8, 2])
    i = 0
    while sum(out) < F:
        out.append(min(pat[i % len(pat)], F - sum(out)))
        i += 1
    return out


def _decode_whole(model, emb, scale):
    """fcb_decode_emb on the whole clip (scale dev [B] or None)."""
    B, F, _ = emb.shape
    out = torch.empty((B, 1, F * model.cfg.hop_length), device="cuda")
    sc = None if scale is None else scale.reshape(-1).contiguous()
    from funcodec_b200.encodec import _ptr
    model._ck(model._lib.fcb_decode_emb(model._h, _ptr(emb.contiguous()), B, F, _ptr(sc), _ptr(out), out.shape[-1],
                                        model._stream()), "fcb_decode_emb")
    return out


def _whole(model, wav):
    r = model.inference(wav, need_recon=False, need_sub_quants=False)
    codes, (quant, scale) = r["code_indices"][0], r["code_embeddings"][0]
    return codes, quant, scale


def _stream_all(model, wav, sched, scale):
    hop = model.cfg.hop_length
    B = wav.shape[0]
    es, ds, de = model.encode_stream(B, scale), model.decode_stream(B, scale), model.decode_stream(B, scale)
    codes, quants, rec_c, rec_e = [], [], [], []
    pos = 0
    for f in sched:
        c, q = es.push(wav[:, pos * hop:(pos + f) * hop])
        codes.append(c)
        quants.append(q)
        rec_c.append(ds.push_codes(c.permute(1, 2, 0)))
        rec_e.append(de.push_emb(q))
        pos += f
    return torch.cat(codes, 2), torch.cat(quants, 1), torch.cat(rec_c, 2), torch.cat(rec_e, 2)


def _check_equivalence(name, use_tc, B, seconds, sched_kind):
    cfg, _, model = _model(name, use_tc)
    hop = cfg.hop_length
    F = int(seconds * cfg.sample_rate) // hop
    wav = _wav(B, F * hop)
    codes, quant, scale = _whole(model, wav)
    sc = scale.reshape(-1) if scale is not None else None
    fmin = cfg.stream_min_first_frames()
    sched = _schedule(sched_kind, F, fmin)
    s_codes, s_quant, s_rec_c, s_rec_e = _stream_all(model, wav, sched, sc)
    assert torch.equal(s_codes, codes), (name, sched_kind, (s_codes != codes).sum().item())
    assert torch.equal(s_quant, quant), (name, sched_kind, (s_quant - quant).abs().max().item())
    rec = _decode_whole(model, quant, sc)
    assert torch.equal(s_rec_e, rec), (name, sched_kind, (s_rec_e - rec).abs().max().item())
    emb = model.inference_decoding(codes.permute(1, 2, 0))["code_embeddings"][0][0]
    rec_c = _decode_whole(model, emb, sc)
    assert torch.equal(s_rec_c, rec_c), (name, sched_kind, (s_rec_c - rec_c).abs().max().item())


@pytest.mark.parametrize("sched_kind", ["ones", "mixed", "single"])
@pytest.mark.parametrize("use_tc", [1, 0], ids=["tc", "simt"])
@pytest.mark.parametrize("name", CAUSAL)
def test_stream_equals_whole_clip(name, use_tc, sched_kind):
    _check_equivalence(name, use_tc, 2, 2.0, sched_kind)


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("name", CAUSAL)
def test_stream_equals_whole_clip_batch_sizes(name, B):
    _check_equivalence(name, 1, B, 1.0, "mixed")


def test_min_first_frames_matches_config():
    for name in CAUSAL:
        cfg, _, model = _model(name)
        assert model.encode_stream(1, torch.ones(1)).min_first_frames == cfg.stream_min_first_frames() == 7


@pytest.mark.parametrize("name", ["soundstream_causal_small", "causal_lstm_small"])
def test_decode_stream_foreign_codes_and_varying_n_q(name):
    """Seeded random tokens (not the encoder's), n_q below the maximum on some calls: the decoder stream equals the whole-clip
    decode of the per-chunk embedding sums (the embedding lookup keeps no state across frames)."""
    cfg, _, model = _model(name)
    B, F = 2, 60
    g = torch.Generator().manual_seed(3)
    tok = torch.randint(0, cfg.codebook_size, (B, F, cfg.num_quantizers), generator=g).cuda()
    sched = _schedule("mixed", F, cfg.stream_min_first_frames())
    nqs = [cfg.num_quantizers if i % 2 == 0 else max(1, cfg.num_quantizers // 2 - i % 3) for i in range(len(sched))]
    one = torch.ones(B, device="cuda")
    ds = model.decode_stream(B, one)
    outs, embs = [], []
    pos = 0
    for f, nq in zip(sched, nqs):
        t = tok[:, pos:pos + f, :nq]
        outs.append(ds.push_codes(t))
        embs.append(model.inference_decoding(t)["code_embeddings"][0][0])
        pos += f
    whole = model.inference_decoding_emb(torch.cat(embs, 1))["recon_speech"]
    assert torch.equal(torch.cat(outs, 2), whole)


def test_stream_isolation_and_reset():
    """A B = 3 stream equals three B = 1 streams; two streams on one handle with interleaved calls equal each run alone;
    reset() reproduces the first run."""
    cfg, _, model = _model("causal_lstm_small")
    hop = cfg.hop_length
    F = 40
    wav = _wav(3, F * hop, seed=21)
    _, _, scale = _whole(model, wav)
    sc = scale.reshape(-1)
    sched = _schedule("mixed", F, cfg.stream_min_first_frames())

    def run(es, x):
        out, pos = [], 0
        for f in sched:
            out.append(es.push(x[:, pos * hop:(pos + f) * hop])[0])
            pos += f
        return torch.cat(out, 2)

    es3 = model.encode_stream(3, sc)
    c3 = run(es3, wav)
    for b in range(3):
        assert torch.equal(run(model.encode_stream(1, sc[b:b + 1]), wav[b:b + 1]), c3[:, b:b + 1])
    es3.reset()
    assert torch.equal(run(es3, wav), c3)
    # interleaved: two streams, alternating calls
    ea = model.encode_stream(3, sc)
    wav_b = _wav(3, F * hop, seed=22)
    _, _, scale_b = _whole(model, wav_b)
    eb = model.encode_stream(3, scale_b.reshape(-1))
    cb_alone = run(model.encode_stream(3, scale_b.reshape(-1)), wav_b)
    outa, outb, pos = [], [], 0
    for f in sched:
        outa.append(ea.push(wav[:, pos * hop:(pos + f) * hop])[0])
        outb.append(eb.push(wav_b[:, pos * hop:(pos + f) * hop])[0])
        pos += f
    assert torch.equal(torch.cat(outa, 2), c3)
    assert torch.equal(torch.cat(outb, 2), cb_alone)


def test_stream_refusals():
    cfg, _, model = _model("soundstream_causal_small")
    hop, fmin = cfg.hop_length, cfg.stream_min_first_frames()
    with pytest.raises(_capi.FcbError, match="causal"):
        _model("soundstream_noncausal_small")[2].encode_stream(1)
    with pytest.raises(_capi.FcbError, match="time-domain"):
        _model("freq_small")[2].decode_stream(1)
    with pytest.raises(_capi.FcbError, match="segment_dur"):
        _model("soundstream_causal_small", segment_dur=1.0, overlap_ratio=0.01)[2].encode_stream(1, torch.ones(1))
    with pytest.raises(_capi.FcbError, match="scale"):
        model.encode_stream(2)
    with pytest.raises(_capi.FcbError, match="scale"):
        model.decode_stream(2)
    es = model.encode_stream(2, torch.ones(2))
    with pytest.raises(_capi.FcbError, match="multiple of the hop"):
        es.push(_wav(2, fmin * hop + 7))
    with pytest.raises(_capi.FcbError, match=f"at least {fmin} frames"):
        es.push(_wav(2, (fmin - 1) * hop))
    with pytest.raises(ValueError, match="clips"):
        es.push(_wav(3, fmin * hop))
    es.push(_wav(2, fmin * hop))            # a refused call leaves the stream usable
    es.push(_wav(2, hop))
    ds = model.decode_stream(2, torch.ones(2))
    bad = torch.zeros((2, fmin, cfg.num_quantizers), dtype=torch.int64)
    bad[1, 3, 0] = cfg.codebook_size
    with pytest.raises(IndexError, match="out of range"):
        ds.push_codes(bad)


def test_causal_lstm_small_whole_clip_against_oracle():
    """No other GPU test covers {weight_norm, causal, SLSTM}: the whole-clip path against the CPU oracle."""
    cfg, sd, model = _model("causal_lstm_small")
    oracle = O.OracleEncodec.from_config(sd, cfg)
    wav = _wav(3, 40 * 25 + 3, seed=7).cpu()
    ora = oracle.inference(wav, want_margin=True)
    r = model.inference(wav, need_recon=True)
    codes = r["code_indices"][0].cpu().numpy()
    res = assert_codes_parity(codes, ora["code_indices"][0].numpy(), ora["margins"].numpy(), 2e-3, what="causal_lstm_small")
    ok = ~(res["first_stage"] >= 0).any(axis=1)
    rec, orec = r["recon_speech"].cpu().numpy(), ora["recon_speech"].numpy()
    for b in np.nonzero(ok)[0]:
        assert np.abs(rec[b] - orec[b]).max() <= 1e-4
