"""CPU ORACLE for the FreqCodec (mag_phase) variant of the hot path -- BASELINE config 4.  TEST INFRASTRUCTURE ONLY.

The checker for the CUDA path of SURVEY.md §8 rows R19-R20: a functional restatement over
torch CPU ops of `FreqCodec._encode_frame / _decode_frame` (mag_phase branches, funcodec/models/codec_freq.py:330-342,
365-373,386 and :406-425,446-448), `SEANetEncoder2d` / `SEANetDecoder2d` (funcodec/models/encoder/seanet_encoder.py:252-363,
funcodec/models/decoder/seanet_decoder.py:244-360) and `SConv2d` / `SConvTranspose2d` / `pad2d` / `unpad2d`
(funcodec/modules/normed_modules/conv.py:102-141,317-447).  Pinned against the unmodified reference by
tools/gen_golden_freq.py -> tests/golden/freq_*.npz (tests/test_oracle_golden_freq.py).

Layouts are the reference's: 2-D activations [B, C, F, T]; embeddings [B, T', D]; codes [n_q, B, T'].
"""
from typing import Dict, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import encodec_oracle as O

EPS_GN = O.EPS_GN


def pad2d_reflect(x, pad_time: Tuple[int, int], pad_freq: Tuple[int, int]):
    """conv.py:102-120 (pad2d, mode='reflect'); F.pad argument order is (time_l, time_r, freq_l, freq_r)."""
    freq_len, time_len = x.shape[-2:]
    max_t, max_f = max(pad_time), max(pad_freq)
    extra_t = max_t - time_len + 1 if time_len <= max_t else 0
    extra_f = max_f - freq_len + 1 if freq_len <= max_f else 0
    x = F.pad(x, (0, extra_t, 0, extra_f))
    padded = F.pad(x, (*pad_time, *pad_freq), mode="reflect")
    return padded[..., : padded.shape[-2] - extra_f, : padded.shape[-1] - extra_t]


def sconv2d(x, p: Dict[str, torch.Tensor], prefix: str, stride=(1, 1), groups: int = None):
    """SConv2d.forward, non-causal (conv.py:342-376) + NormConv2d (conv.py:180-184): frequency axis gets no extra padding."""
    w = p[prefix + ".conv.conv.weight"]
    b = p[prefix + ".conv.conv.bias"]
    if groups is None:                            # nn.Conv2d weight is [C_out, C_in / groups, kf, kt] (conv_group_ratio > 0)
        groups = x.shape[1] // w.shape[1]
    kf, kt = w.shape[-2:]
    sf, st = stride
    pt_f = (kf - 1) - (sf - 1)
    pt_t = (kt - 1) - (st - 1)
    extra_t = O.extra_padding_for_conv1d(x.shape[-1], kt, st, pt_t)
    f_after = pt_f // 2
    f_before = pt_f - f_after
    t_after = pt_t // 2
    t_before = pt_t - t_after + extra_t          # NB: the reference adds the extra padding on the LEFT in 2-D (:368)
    x = pad2d_reflect(x, (t_before, t_after), (f_before, f_after))
    y = F.conv2d(x, w, b, stride=(sf, st), groups=groups)
    return F.group_norm(y, 1, p[prefix + ".conv.norm.weight"], p[prefix + ".conv.norm.bias"], EPS_GN)


def sconvtr2d(x, p: Dict[str, torch.Tensor], prefix: str, stride, out_padding=((0, 0), (0, 0)), groups: int = None):
    """SConvTranspose2d.forward, non-causal (conv.py:407-447): convtr -> GroupNorm -> unpad2d with out_padding."""
    w = p[prefix + ".convtr.convtr.weight"]
    b = p[prefix + ".convtr.convtr.bias"]
    if groups is None:                            # nn.ConvTranspose2d weight is [C_in, C_out / groups, kf, kt]
        groups = b.shape[0] // w.shape[1]
    kf, kt = w.shape[-2:]
    sf, st = stride
    y = F.conv_transpose2d(x, w, b, stride=(sf, st), groups=groups)
    y = F.group_norm(y, 1, p[prefix + ".convtr.norm.weight"], p[prefix + ".convtr.norm.bias"], EPS_GN)
    pf, pt = kf - sf, kt - st
    pf_r, pt_r = pf // 2, pt // 2
    pf_l, pt_l = pf - pf_r, pt - pt_r
    (fo_l, fo_r), (to_l, to_r) = out_padding
    tl, tr = max(pt_l - to_l, 0), max(pt_r - to_r, 0)
    fl, fr = max(pf_l - fo_l, 0), max(pf_r - fo_r, 0)
    return y[..., fl: y.shape[-2] - fr, tl: y.shape[-1] - tr]


def resblock2d(x, p, prefix: str):
    """SEANetResnetBlock2d.forward (seanet_encoder.py:188-237), true_skip=False; conv groups follow the weight shapes."""
    h = sconv2d(O.elu(x), p, prefix + ".block.1")
    h = sconv2d(O.elu(h), p, prefix + ".block.3")
    return sconv2d(x, p, prefix + ".shortcut") + h


def seanet_encoder2d(x, p, ratios: Sequence[Tuple[int, int]], lstm_layers: int = 2):
    """SEANetEncoder2d.forward: x [B, C_in, F, T] -> [B, T', D].  Encoder applies the ratios reversed (:288)."""
    h = sconv2d(x, p, "model.0")
    n = 1
    for fr, tr in reversed(list(ratios)):
        h = resblock2d(h, p, f"model.{n}")
        h = sconv2d(O.elu(h), p, f"model.{n + 2}", stride=(fr, tr))
        n += 3
    h = torch.squeeze(h, dim=2)            # ReshapeModule(dim=2) (:326)
    n += 1
    if lstm_layers > 0:
        h = O.slstm(h, p, f"model.{n}", lstm_layers)
        n += 1
    h = O.sconv1d(O.elu(h), p, f"model.{n + 1}")
    return h.permute(0, 2, 1)


def seanet_decoder2d(z, p, ratios: Sequence[Tuple[int, int]], lstm_layers: int = 2, last_out_padding=((0, 1), (0, 0))):
    """SEANetDecoder2d.forward: z [B, T', D] -> [B, C_out, F, T]."""
    h = O.sconv1d(z.permute(0, 2, 1), p, "model.0")
    n = 1
    if lstm_layers > 0:
        h = O.slstm(h, p, "model.1", lstm_layers)
        n = 2
    h = torch.unsqueeze(h, dim=2)          # decoder's ReshapeModule (seanet_decoder.py:235-241)
    n += 1
    ratios = list(ratios)
    for i, (fr, tr) in enumerate(ratios):
        op = last_out_padding if i == len(ratios) - 1 else ((0, 0), (0, 0))
        h = sconvtr2d(O.elu(h), p, f"model.{n + 1}", (fr, tr), op)
        h = resblock2d(h, p, f"model.{n + 2}")
        n += 3
    return sconv2d(O.elu(h), p, f"model.{n + 1}")


class OracleFreqCodec:
    """FreqCodec.inference (codec_freq.py:668-716) for codec_domain = ['mag_phase', 'mag_phase']."""

    def __init__(self, state_dict, ratios, sample_rate: int = 16000, lstm_layers: int = 2, n_fft: int = 512,
                 hop: int = 160, audio_normalize: bool = True, dtype=torch.float32):
        sd = {k: v.detach().to("cpu", dtype) if v.is_floating_point() else v.detach().cpu() for k, v in state_dict.items()}
        self.enc = O.sub_dict(sd, "encoder.")
        self.dec = O.sub_dict(sd, "decoder.")
        self.embed = sd["quantizer.rq.model.embed"]
        self.ratios = [tuple(r) for r in ratios]
        self.lstm_layers = lstm_layers
        self.sample_rate = sample_rate
        self.n_fft, self.hop = n_fft, hop
        self.audio_normalize = audio_normalize
        self.dtype = dtype
        self.window = torch.hann_window(n_fft, dtype=dtype)   # torchaudio.transforms.Spectrogram default window

    def stft(self, x_bl):
        return torch.stft(x_bl, self.n_fft, self.hop, self.n_fft, self.window, center=True, pad_mode="reflect",
                          normalized=False, onesided=True, return_complex=True)

    def istft(self, spec):
        return torch.istft(spec, self.n_fft, self.hop, self.n_fft, self.window, center=True, normalized=False,
                           onesided=True, length=None)

    def encode_frame(self, x_b1l):
        """codec_freq.py:330-342 + mag_phase branch :365-373."""
        scale = None
        if self.audio_normalize:
            mono = x_b1l.mean(dim=1, keepdim=True)
            scale = 1e-8 + mono.pow(2).mean(dim=2, keepdim=True).sqrt()
            x_b1l = x_b1l / scale
            scale = scale.view(-1, 1)
        xc = self.stft(x_b1l.squeeze(1))
        mag = torch.abs(xc)
        log_mag = torch.log(torch.clamp(mag, min=1e-6))
        phase = xc / torch.clamp(mag, min=1e-6)
        feats = torch.stack([log_mag, phase.real, phase.imag], dim=1)
        return seanet_encoder2d(feats, self.enc, self.ratios, self.lstm_layers), scale, feats

    def decode_frame(self, emb_btd, scale):
        """codec_freq.py:406-425 (mag_phase) + :446-448."""
        out = seanet_decoder2d(emb_btd, self.dec, self.ratios, self.lstm_layers)
        mag = F.softplus(out[:, 0])
        spec = mag * torch.complex(out[:, 1], out[:, 2])
        wav = self.istft(spec).unsqueeze(1)
        if scale is not None:
            wav = wav * scale.view(-1, 1, 1)
        return wav

    @torch.no_grad()
    def inference(self, speech, need_recon=True, bit_width=None, use_scale=True, want_margin=False):
        speech = speech.to(self.dtype)
        if speech.dim() == 2:
            speech = speech.unsqueeze(1)
        emb, scale, feats = self.encode_frame(speech)
        n_q_max, bins, _ = self.embed.shape
        hop = self.hop * int(torch.tensor([r[1] for r in self.ratios]).prod())          # samples per codec frame
        n_q = O.num_quantizers_for_bandwidth(n_q_max, bins, self.sample_rate, hop, bit_width)
        quant, codes, sub, margins = O.rvq_forward(emb.permute(0, 2, 1), self.embed, min(n_q, n_q_max), want_margin)
        quant_btd = quant.permute(0, 2, 1)
        recon = None
        if need_recon:
            recon = self.decode_frame(quant_btd, scale if use_scale else None)[:, :, : speech.shape[-1]]
        return dict(recon_speech=recon, code_indices=[codes], code_embeddings=[(quant_btd, scale if use_scale else None)],
                    sub_quants=[sub], encoder_out=emb, features=feats, margins=margins)
