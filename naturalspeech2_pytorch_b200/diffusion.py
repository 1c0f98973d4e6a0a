"""`NaturalSpeech2`: the latent-diffusion wrapper around the denoiser, with the call signatures of
naturalspeech2_pytorch.NaturalSpeech2 (ns2.py:1160-1684): `forward` (training loss), `sample`, `ddim_sample`.

Scope (SURVEY section 8): the per-timestep path — schedules, q-sample, v-target, per-sample MSE, min-SNR
weight, the DDIM update and classifier-free guidance — runs on the sm_90a kernels (`ops.q_sample`,
`Model.forward`, `ops.mse_rows`, `ops.ddim_step`, `ops.cfg_combine`).  The once-per-sample conditioning encoders
of the reference (PhonemeEncoder, SpeechPromptEncoder, DurationPitchPredictor, Aligner; ns2.py:228-527,
aligner.py) are out of scope: for a conditional model pass their outputs directly (`prompt_enc=`, `cond=`) or
give a `conditioner` callable that produces them (e.g. the reference modules, see INTEGRATION.md).

`forward` returns a differentiable loss: the denoiser records one autograd node (training.DenoiserFunction), and with
rvq_cross_entropy_loss_weight > 0 the RVQ cross-entropy term records another (`XStartCrossEntropyFunction`) whose
backward hands d pred to the denoiser's, as the reference's autograd does.
"""
from __future__ import annotations

import math
from functools import partial
from typing import Callable, Optional

import torch
from torch import nn

from . import ops
from .codec import EncodecRVQ, codes_past_lengths
from .seanet import frame_lengths
from .model import Model


def _exists(v):
    return v is not None


# ---- noise schedules (ns2.py:1133-1156); tiny (B,)-sized host-side torch math ----
def simple_linear_schedule(t, clip_min=1e-9):
    return (1 - t).clamp(min=clip_min)


def cosine_schedule(t, start=0, end=1, tau=1, clip_min=1e-9):
    """ns2.py:1136-1142 on tensors (the reference's `math.cos` raises on them, SURVEY T12).  The cosine is clamped at
    0 before the power: in fp32 cos(pi/2) is -4.4e-8, which a fractional power (non-integer 2 tau) turns into NaN."""
    power = 2 * tau
    v_start = math.cos(start * math.pi / 2) ** power
    v_end = math.cos(end * math.pi / 2) ** power
    output = torch.cos((t * (end - start) + start) * math.pi / 2).clamp(min=0) ** power
    output = (v_end - output) / (v_end - v_start)
    return output.clamp(min=clip_min)


def sigmoid_schedule(t, start=-3, end=3, tau=1, clamp_min=1e-9):
    v_start = torch.tensor(start / tau).sigmoid()
    v_end = torch.tensor(end / tau).sigmoid()
    gamma = (-((t * (end - start) + start) / tau).sigmoid() + v_end) / (v_end - v_start)
    return gamma.clamp_(min=clamp_min, max=1.)


def gamma_to_alpha_sigma(gamma, scale=1):
    return torch.sqrt(gamma) * scale, torch.sqrt(1 - gamma)


class NaturalSpeech2(nn.Module):
    def __init__(self, model: Model, codec=None, *, tokenizer=None, target_sample_hz=None, timesteps=1000,
                 use_ddim=True, noise_schedule="sigmoid", objective="v", schedule_kwargs: dict = dict(),
                 time_difference=0., min_snr_loss_weight=True, min_snr_gamma=5, train_prob_self_cond=0.9,
                 rvq_cross_entropy_loss_weight=0., scale=1., duration_loss_weight=1., pitch_loss_weight=1.,
                 conditioner: Optional[Callable] = None, cuda_graphs: bool = True, **conditioning_kwargs):
        super().__init__()
        if not isinstance(model, Model):
            raise TypeError("model must be a naturalspeech2_pytorch_b200.Model")
        self.conditional = model.condition_on_prompt
        self.model = model
        self.codec = codec
        assert _exists(codec) or _exists(target_sample_hz)  # ns2.py:1207
        self.target_sample_hz = target_sample_hz
        self.seq_len_multiple_of = None
        if _exists(codec):
            self.target_sample_hz = codec.target_sample_hz
            self.seq_len_multiple_of = codec.seq_len_multiple_of
        assert not _exists(codec) or model.dim == codec.codebook_dim, \
            f"transformer model dimension {model.dim} must be equal to codec dimension {codec.codebook_dim}"
        self.dim = codec.codebook_dim if _exists(codec) else model.dim
        assert objective in {"x0", "eps", "v"}
        self.objective = objective
        sched = {"linear": simple_linear_schedule, "cosine": cosine_schedule, "sigmoid": sigmoid_schedule}
        if noise_schedule not in sched:
            raise ValueError(f"invalid noise schedule {noise_schedule}")
        assert scale <= 1, "scale must be less than or equal to 1"
        self.scale = scale
        self.gamma_schedule = partial(sched[noise_schedule], **schedule_kwargs)
        self.timesteps = timesteps
        self.use_ddim = use_ddim
        self.time_difference = time_difference
        self.train_prob_self_cond = train_prob_self_cond
        self.min_snr_loss_weight = min_snr_loss_weight
        self.min_snr_gamma = min_snr_gamma
        self.rvq_cross_entropy_loss_weight = rvq_cross_entropy_loss_weight
        self.duration_loss_weight, self.pitch_loss_weight = duration_loss_weight, pitch_loss_weight   # ns2.py:1193-1194
        self.conditioner = conditioner
        self.cuda_graphs = cuda_graphs  # sampling loop: replay one captured CUDA graph per sampling step
        self.conditioning_kwargs = conditioning_kwargs  # accepted for signature parity (encoder hyper-parameters)

    @property
    def device(self):
        return next(self.model.parameters()).device

    def get_sampling_timesteps(self, batch, *, device):
        """ns2.py:1303-1308."""
        times = torch.linspace(1., 0., self.timesteps + 1, device=device)
        times = times[None].expand(batch, -1)
        times = torch.stack((times[:, :-1], times[:, 1:]), dim=0)
        return times.unbind(dim=-1)

    # ------------------------------------------------------------------------------------------
    # sampling
    # ------------------------------------------------------------------------------------------
    def _schedule_tables(self, batch, device):
        """(times (T, B), coef (T, 4, B) = alpha, sigma, alpha_next, sigma_next) for every sampling step, computed with
        the reference's own element-wise formulas (ns2.py:1303-1308, 1396-1404), so the values are bit-identical to
        the per-step tensors the reference builds."""
        t_all = torch.linspace(1., 0., self.timesteps + 1, device=device)
        gamma = self.gamma_schedule(t_all)
        alpha, sigma = gamma_to_alpha_sigma(gamma, self.scale)
        coef = torch.stack((alpha[:-1], sigma[:-1], alpha[1:], sigma[1:]), dim=1)      # (T, 4)
        times = t_all[:-1, None].expand(-1, batch).contiguous()
        return times, coef[:, :, None].expand(-1, -1, batch).contiguous()

    def _sampler_entry(self, shape, conditioning, cond_scale, device, lens=None):
        """One captured CUDA graph = one whole sampling step: denoiser forward(s), guidance combine, DDIM update of the
        static latent buffer.  Keyed on shapes (and on whether latent lengths are given) only; conditioning and the
        lengths are copied into static buffers.  It replays on the model's workspace, so the model caches it."""
        guided = self.conditional and cond_scale != 1.
        cond_sig = None
        if conditioning is not None:
            cond_sig = tuple(tuple(v.shape) for v in conditioning.values() if torch.is_tensor(v))
        key = ("sample", tuple(shape), cond_sig, float(cond_scale) if guided else None, self.objective,
               lens is not None, str(device))
        model, B = self.model, shape[0]

        def build(cond):
            x = torch.empty(shape, device=device, dtype=torch.float32)
            ts = torch.zeros(B, device=device, dtype=torch.float32)
            coef = torch.ones(4, B, device=device, dtype=torch.float32)
            v0 = torch.empty_like(x)
            v1 = torch.empty_like(x) if guided else None
            p_cond = 0. if self.conditional else None
            static_lens = None if lens is None else lens.clone()

            def step():
                model._forward_impl(x, ts, cond_drop_prob=p_cond, _conditioning=cond, out=v0, lengths=static_lens)
                if guided:   # classifier-free guidance (ns2.py:914-927): conditional + null forward, lerp
                    model._forward_impl(x, ts, cond_drop_prob=1., _conditioning=cond, out=v1, lengths=static_lens)
                    ops.cfg_combine(v0, v1, cond_scale, v0)
                ops.ddim_step(x, v0, coef[0], coef[1], coef[2], coef[3], objective=self.objective)

            x.normal_()
            return {"x": x, "ts": ts, "coef": coef, "v": (v0, v1), "lens": static_lens}, step

        entry = model._captured(key, model._ws_key(B, shape[1], device), conditioning, build)
        if lens is not None:
            entry["lens"].copy_(lens)
        return entry

    @torch.no_grad()
    def ddim_sample(self, shape, prompt=None, time_difference=None, cond_scale=1., cond=None, *, noise=None,
                    prompt_lens=None, cond_lens=None, latent_lens=None):
        """ns2.py:1379-1431.  `noise` (optional) fixes the initial latent instead of drawing it.
        (`time_difference` only shifts a value the reference never reads again, ns2.py:1404-1406.)
        prompt_lens / cond_lens: per-sample lengths of the prompt and the condition (Model.precompute_conditioning).
        latent_lens: per-sample latent lengths (`Model.forward`'s `lengths`); the result is zero past them."""
        batch, device = shape[0], self.device
        lens = None
        if latent_lens is not None:
            lens = self.model._latent_lens(latent_lens, torch.empty(shape[:2], device=device))
        # a dense, row-major copy: the eager loop updates it in place with ops.ddim_step, which reads flat arrays
        audio = torch.randn(shape, device=device) if noise is None else \
            noise.to(device).float().clone(memory_format=torch.contiguous_format)
        conditioning = None
        if self.conditional:
            assert _exists(prompt) and _exists(cond)
            # timestep-invariant work (perceiver, prompt FiLM vector, aligned-condition projection) once
            conditioning = self.model.precompute_conditioning(prompt, cond, shape[1], prompt_lens=prompt_lens,
                                                              cond_lens=cond_lens)
        times_tab, coef_tab = self._schedule_tables(batch, device)
        if self.cuda_graphs and audio.is_cuda and self.model._prof is None:
            entry = self._sampler_entry(shape, conditioning, cond_scale, device, lens)
            entry["x"].copy_(audio)
            for i in range(self.timesteps):
                entry["ts"].copy_(times_tab[i])
                entry["coef"].copy_(coef_tab[i])
                entry["graph"].replay()
            audio = entry["x"].clone()
            return audio if lens is None else ops.mask_rows(audio, lens)
        extra = {} if lens is None else {"lengths": lens}
        for i in range(self.timesteps):
            if self.conditional:
                v = self.model.forward_with_cond_scale(audio, times_tab[i], cond_scale=cond_scale,
                                                       _conditioning=conditioning, **extra)
            else:
                v = self.model.forward_with_cond_scale(audio, times_tab[i], cond_scale=cond_scale, **extra)
            c = coef_tab[i]
            ops.ddim_step(audio, v, c[0], c[1], c[2], c[3], objective=self.objective)
        return audio if lens is None else ops.mask_rows(audio, lens)

    def _encodes_lengths(self) -> bool:
        """Whether the codec encodes a padded batch of waveforms with per-sample lengths (an EncodecRVQ with an
        encoder, e.g. SEANetEncoder)."""
        return isinstance(self.codec, EncodecRVQ) and self.codec.encoder is not None

    def _encode_prompt(self, prompt, prompt_lens):
        """A raw-audio prompt batch (B, T) with per-sample lengths (frames) -> its latents (B, T // hop, dim), each
        sample's bit-identical to encoding its waveform alone and zero past its length.  Anything else is returned
        as it is."""
        if prompt is not None and prompt.ndim == 2 and prompt_lens is not None and self._encodes_lengths():
            prompt, _, _ = self.codec(prompt, return_encoded=True, lengths=prompt_lens)
        return prompt

    def _check_latent_lens_training(self, audio, codes, latent_lens):
        """Refuse, before any launch, what `forward(latent_lens=)` does not support."""
        if audio.ndim == 2:
            if not self._encodes_lengths():
                raise ValueError("latent_lens needs encoded latents (B, N, dim) unless the codec is an EncodecRVQ with "
                                 "an encoder: this codec's encoder takes no lengths")
            frame_lengths(latent_lens, audio.shape[0], audio.shape[-1] // self.codec.seq_len_multiple_of,
                          device=audio.device)
        if self.rvq_cross_entropy_loss_weight != 0 and (codes is not None or audio.ndim == 2) and \
                not isinstance(self.codec, EncodecRVQ):
            raise NotImplementedError("latent_lens with the RVQ cross-entropy term needs an EncodecRVQ codec (the -1 "
                                      "targets past each length are its ignore_index)")
        cn = self.conditioner
        if cn is not None and getattr(cn, "train_duration_pitch", False):
            raise NotImplementedError("latent_lens with train_duration_pitch is not supported")
        if cn is not None and isinstance(cn, torch.nn.Module) and cn.training and any(
                getattr(m, "train_dropout", False) for m in cn.modules()):
            raise NotImplementedError("latent_lens with training dropout (train_dropout) is not supported")

    def process_prompt(self, prompt=None):
        """ns2.py:1433-1447."""
        if not _exists(prompt):
            return None
        assert self.model.condition_on_prompt
        if prompt.ndim == 2:
            assert _exists(self.codec), "codec must be passed in if one were to train on raw prompt"
            with torch.no_grad():
                prompt, _, _ = self.codec(prompt, curtail_from_left=True, return_encoded=True)
        return prompt

    @torch.no_grad()
    def sample(self, *, length, prompt=None, batch_size=1, cond_scale=1., text=None, text_lens=None,
               prompt_enc=None, cond=None, noise=None, prompt_lens=None, phoneme_lens=None, cond_lens=None,
               latent_lens=None):
        """ns2.py:1457-1501.  Conditional models need (`prompt_enc`, `cond`) or a `conditioner`.
        `text_lens` is accepted and ignored, as in the reference.  A batch of prompts and texts of different lengths,
        padded at their ends, is sampled as if each sample ran alone with `prompt_lens` (prompt latent frames) and
        `phoneme_lens` (phonemes), given to the conditioner, whose condition lengths then follow; with precomputed
        `prompt_enc=` / `cond=` pass `prompt_lens` and `cond_lens` (condition frames) instead.  With lengths the
        prompt is encoded latents (B, Np, dim), or raw audio (B, T) with `prompt_lens` when the codec is an EncodecRVQ
        with an encoder: sample b's prompt is then prompt[b, :prompt_lens[b] * hop] (at least 7 frames), encoded as if
        alone (`EncodecRVQ.forward(lengths=)`).  Other raw-audio prompts would be curtailed by the batch's length.

        latent_lens (B,): sample b is `latent_lens[b]` latent frames long (`length` stays the padded length, at most 64
        samples): each returned latent equals sampling that sample alone with length=latent_lens[b] and the first
        latent_lens[b] frames of its noise, bit for bit, and is zero past it.  The denoiser skips the 128-frame tiles
        wholly past each length.  With a codec, each waveform is zero past latent_lens[b] * hop samples; the SEANet
        decoder is causal, so its prefix is the sample's waveform decoded alone provided latent_lens[b] >= 7 frames
        (shorter inputs fall under Encodec's short-input padding rule when decoded alone, which a batch cannot
        reproduce)."""
        if self.use_ddim is False:
            raise NotImplementedError("ddpm_sample is dead code in the reference (NameError: expm1, SURVEY T8)")
        ragged = prompt_lens is not None or phoneme_lens is not None or cond_lens is not None
        if ragged and not self.conditional:
            raise ValueError("prompt_lens / phoneme_lens / cond_lens apply to conditional models")
        if self.conditional:
            prompt = self._encode_prompt(prompt, prompt_lens)
            if not (_exists(prompt_enc) and _exists(cond)):
                if not _exists(self.conditioner):
                    raise NotImplementedError(
                        "conditional sampling needs prompt_enc= and cond= (outputs of the reference's "
                        "SpeechPromptEncoder / duration-pitch expansion) or a `conditioner` callable")
                if not ragged:
                    prompt_enc, cond = self.conditioner(prompt=self.process_prompt(prompt), text=text,
                                                        text_lens=text_lens, mode="sample")
                else:
                    if cond_lens is not None:
                        raise ValueError("cond_lens goes with precomputed prompt_enc= / cond=; the conditioner "
                                         "computes it from phoneme_lens")
                    if prompt is None or prompt.ndim != 3:
                        raise ValueError("with prompt_lens / phoneme_lens the prompt must be encoded latents (B, Np, dim): "
                                         "a raw-audio prompt is curtailed from the left by the batch's length")
                    prompt_enc, cond, cond_lens = self.conditioner(
                        prompt=prompt, text=text, text_lens=text_lens, mode="sample", prompt_lens=prompt_lens,
                        phoneme_lens=phoneme_lens)
            elif phoneme_lens is not None:
                raise ValueError("phoneme_lens goes to the conditioner; with prompt_enc= / cond= pass cond_lens")
            batch_size = prompt_enc.shape[0]
        if latent_lens is not None and prompt is not None and prompt.ndim == 2:
            raise ValueError("latent_lens needs an encoded prompt (B, Np, dim) or prompt_enc=: a raw-audio prompt is "
                             "curtailed from the left by the batch's length")
        audio = self.ddim_sample((batch_size, length, self.dim), prompt=prompt_enc, cond=cond,
                                 cond_scale=cond_scale, noise=noise, prompt_lens=prompt_lens, cond_lens=cond_lens,
                                 latent_lens=latent_lens)
        if _exists(self.codec):
            audio = self.codec.decode(audio)
            if audio.ndim == 3 and audio.shape[1] == 1:
                audio = audio[:, 0]
            if latent_lens is not None and audio.ndim == 2:   # a waveform: zeros past each sample's frames
                lens = self.model._latent_lens(latent_lens, torch.empty(batch_size, length, device=audio.device))
                hop = audio.shape[-1] // length
                if hop * length != audio.shape[-1]:
                    raise ValueError(f"latent_lens: the codec returned {audio.shape[-1]} samples for {length} frames")
                audio = ops.mask_rows(audio.contiguous().view(batch_size, length, hop), lens).view(batch_size, -1)
        return audio

    # ------------------------------------------------------------------------------------------
    # training loss (differentiable: `loss.backward()` runs the hand-written backward kernels)
    # ------------------------------------------------------------------------------------------
    def forward(self, audio, text=None, text_lens=None, mel=None, mel_lens=None, codes=None, prompt=None,
                pitch=None, *args, prompt_enc=None, cond=None, times=None, noise=None, duration=None, prompt_lens=None,
                phoneme_lens=None, latent_lens=None, **kwargs):
        """ns2.py:1503-1684 -> scalar diffusion loss (the only term the reference returns, SURVEY T11).
        Extra keyword-only arguments: `prompt_enc`/`cond` (precomputed conditioning), `times`/`noise`
        (inject the two random draws of ns2.py:1621,1625 — used by the parity tests) and `duration` (per-phoneme frame
        counts, handed to the conditioner only when given: encoders.Conditioner takes them in place of an aligner).
        A conditioner that returns (prompt_enc, cond, duration_loss, pitch_loss) (encoders.Conditioner with
        train_duration_pitch=True) adds duration_loss_weight * duration_loss + pitch_loss_weight * pitch_loss to the
        returned loss, the `aux_loss` of ns2.py:1600-1602 that the reference adds at 1684.
        A batch of prompts and texts of different lengths, padded at their ends, trains as if each sample ran alone with
        `prompt_lens` (prompt latent frames) and `phoneme_lens` (phonemes), given to the conditioner, and prompt_lens to
        the model; with precomputed `prompt_enc=` / `cond=` only prompt_lens (to the model).  A raw-audio prompt (B, T)
        with prompt_lens is encoded with those lengths when the codec is an EncodecRVQ with an encoder, as in `sample`.
        The latents and pitch share one length.  Each sample's MSE row is then that of the sample alone; the loss, as in
        the reference, is mean(mse) * mean(weight) over the batch (ns2.py:1651-1666), not the mean of the per-sample
        losses.

        latent_lens (B,): sample b's latents are audio[b, :latent_lens[b]] (encoded latents, padded at the end, at most
        64 samples); its MSE row is the mean over those frames only, bit-identical to the sample alone, and its
        gradients are those of the sample alone (rows past the length add exact zeros).  Combines with prompt_lens /
        phoneme_lens.  Raw audio (B, T) takes latent_lens in frames when the codec is an EncodecRVQ with an encoder:
        sample b is audio[b, :latent_lens[b] * hop] (at least 7 frames), encoded as if alone
        (`EncodecRVQ.forward(lengths=)`), and the latents (B, T // hop, dim) then take the path above.  With the RVQ
        cross-entropy term (EncodecRVQ codecs only) the targets past each length are -1, the reference's ignore_index,
        so each stage's term is the mean over the batch's valid frames.  Not with train_duration_pitch or training
        dropout."""
        is_raw_audio = audio.ndim == 2
        aux_loss = None
        if latent_lens is not None:
            self._check_latent_lens_training(audio, codes, latent_lens)
        ragged = prompt_lens is not None or phoneme_lens is not None
        if ragged and not self.conditional:
            raise ValueError("prompt_lens / phoneme_lens apply to conditional models")
        if self.conditional and not (_exists(prompt_enc) and _exists(cond)):
            prompt = self._encode_prompt(prompt, prompt_lens)
            if not _exists(self.conditioner):
                raise NotImplementedError(
                    "conditional training needs prompt_enc= and cond= or a `conditioner` callable (the "
                    "reference's encoders + aligner are outside the accelerated path)")
            extra = {} if duration is None else {"duration": duration}
            if ragged:
                if prompt is None or prompt.ndim != 3:
                    raise ValueError("with prompt_lens / phoneme_lens the prompt must be encoded latents (B, Np, dim): "
                                     "a raw-audio prompt is curtailed from the left by the batch's length")
                extra.update(prompt_lens=prompt_lens, phoneme_lens=phoneme_lens)
            out = self.conditioner(audio=audio, text=text, text_lens=text_lens, mel=mel, mel_lens=mel_lens,
                                   prompt=self.process_prompt(prompt), pitch=pitch, mode="train", **extra)
            prompt_enc, cond = out[:2]
            if len(out) == 4:   # the duration / pitch predictor's L1 losses (ns2.py:1587-1602)
                aux_loss = self.duration_loss_weight * out[2] + self.pitch_loss_weight * out[3]
        elif phoneme_lens is not None:
            raise ValueError("phoneme_lens goes to the conditioner; with prompt_enc= / cond= pass prompt_lens only")
        assert not (is_raw_audio and not _exists(self.codec)), \
            "codec must be passed in if one were to train on raw audio"
        if is_raw_audio:
            extra = {} if latent_lens is None else {"lengths": latent_lens}
            audio, codes, _ = self.codec(audio, return_encoded=True, **extra)
        audio = audio.float().contiguous()
        batch, n, d = audio.shape
        device = self.device
        assert d == self.dim, f"codec codebook dimension {d} must match model dimensions {self.dim}"
        if times is None:
            times = torch.zeros((batch,), device=device).float().uniform_(0, 1.)
        if noise is None:
            noise = torch.randn_like(audio)
        times = times.to(device).float()
        noise = noise.to(device).float().contiguous()
        gamma = self.gamma_schedule(times)
        alpha, sigma = gamma_to_alpha_sigma(gamma, self.scale)
        alpha, sigma = alpha.contiguous(), sigma.contiguous()
        noised = torch.empty_like(audio)
        target = torch.empty_like(audio)
        ops.q_sample(audio, noise, alpha, sigma, noised, target, objective=self.objective)  # ns2.py:1631-1644
        lens = {} if prompt_lens is None else {"prompt_lens": prompt_lens}
        llens = None
        if latent_lens is not None:
            llens = self.model._latent_lens(latent_lens, audio)
            lens["lengths"] = llens
        pred = self.model(noised, times, prompt=prompt_enc, cond=cond, **lens)  # ns2.py:1635
        if pred.requires_grad:
            from .training import MseRowsFunction
            loss = MseRowsFunction.apply(pred, target, *(() if llens is None else (llens,)))   # ns2.py:1646-1647
        else:
            loss = ops.mse_rows(pred, target, torch.empty(batch, device=device), lens=llens)
        # min-SNR weight on (B,)-sized tensors, with the reference's exact broadcasting (ns2.py:1651-1666):
        # loss is (B,), loss_weight is (B,1,1) -> the product is (B,1,B) before .mean()
        a3, s3 = alpha.view(-1, 1, 1), sigma.view(-1, 1, 1)
        snr = (a3 * a3) / (s3 * s3)
        clipped = snr.clone()
        if self.min_snr_loss_weight:
            clipped.clamp_(max=self.min_snr_gamma)
        if self.objective == "eps":       # ns2.py:1657-1664
            loss_weight = clipped / snr
        elif self.objective == "x0":
            loss_weight = clipped
        else:
            loss_weight = clipped / (snr + 1)
        loss = (loss * loss_weight).mean()
        if self.rvq_cross_entropy_loss_weight == 0 or not _exists(codes):   # ns2.py:1670-1671
            return loss if aux_loss is None else loss + aux_loss
        # cross entropy of the predicted x_start against the codec's codes (ns2.py:1673-1684); with latent_lens the
        # targets past each length are -1 (ignored) and x_start is zero there
        if llens is not None:
            codes = codes_past_lengths(codes.reshape(batch, n, -1).to(torch.int64), llens.tolist())
        if pred.requires_grad and isinstance(self.codec, EncodecRVQ):
            ce_loss = XStartCrossEntropyFunction.apply(pred, audio, alpha, sigma, self.codec, codes, self.objective,
                                                       llens)
        else:   # no gradient wanted, or a codec other than EncodecRVQ (its `rq` gets a constant x_start)
            x_start = torch.empty_like(audio)
            ops.x_start_from_pred(audio, pred.detach(), alpha, sigma, x_start, objective=self.objective)
            if llens is not None:
                ops.mask_rows(x_start, llens)
            _, ce_loss = self.codec.rq(x_start, codes)
        loss = loss + self.rvq_cross_entropy_loss_weight * ce_loss
        return loss if aux_loss is None else loss + aux_loss

    p_losses = forward  # the name BASELINE.json's north_star uses; the reference inlines it in forward


def x_start_pred_coef(alpha: torch.Tensor, sigma: torch.Tensor, objective: str) -> Optional[torch.Tensor]:
    """Per-sample d x_start / d pred of ns2.py:1673-1680 ((B,)-sized glue): -sigma (v), -sigma / max(alpha, 1e-10)
    (eps, safe_div ns2.py:1122-1123), None = 1 (x0)."""
    if objective == "v":
        return (-sigma).contiguous()
    if objective == "eps":
        return (-sigma / alpha.clamp(min=1e-10)).contiguous()
    return None


class XStartCrossEntropyFunction(torch.autograd.Function):
    """ns2.py:1673-1682 as one autograd node: x_start from the model output, then `codec.rq`'s CE loss.  The forward
    launches the kernels of the no-grad path (ops.x_start_from_pred, the codec's own codes, ops.rvq_ce), so the loss
    is bit-identical to it; the backward is one `ops.rvq_ce_bwd` call whose per-sample row scale is d x_start / d pred,
    so it returns d pred directly."""

    @staticmethod
    def forward(ctx, pred, audio, alpha, sigma, codec, codes, objective, lens=None):
        x_start = torch.empty_like(audio)
        ops.x_start_from_pred(audio, pred.detach(), alpha, sigma, x_start, objective=objective)
        if lens is not None:   # latent lengths: frames past them (targets -1) are zero, whatever the padding held
            ops.mask_rows(x_start, lens)
        ctx.lens = lens
        flat = x_start.view(-1, 128)
        tgt = codes.reshape(-1, codec.num_quantizers).to(torch.int64).contiguous()
        prep = codec._prep()
        own = ops.rvq_encode(flat, codec.codebooks, prep)
        loss = ops.rvq_ce(flat, codec.codebooks, prep[1], own, tgt)
        coef = x_start_pred_coef(alpha, sigma, objective)
        ctx.save_for_backward(flat, codec.codebooks, prep[1], own, tgt, coef)
        ctx.rows_per_sample = audio.shape[1]
        return loss

    @staticmethod
    def backward(ctx, d_loss):
        flat, codebooks, cn2, own, tgt, coef = ctx.saved_tensors
        d_pred = ops.rvq_ce_bwd(flat, codebooks, cn2, own, tgt, d_loss.float().reshape(1).contiguous(), row_scale=coef,
                                rows_per_sample=ctx.rows_per_sample)
        n = ctx.rows_per_sample
        d_pred = d_pred.view(flat.shape[0] // n, n, 128)
        if ctx.lens is not None:   # frames whose targets are all -1 get nothing; written as +0 whatever the row scale
            ops.mask_rows(d_pred, ctx.lens)
        return d_pred, None, None, None, None, None, None, None
