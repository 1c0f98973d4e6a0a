"""Encodec's 24 kHz SEANet codec on sm_90a, both directions: `SEANetDecoder` is the `decoder` of `EncodecRVQ` (75 Hz
latents -> 24 kHz audio, what `codec.decode(audio)` runs at the end of `NaturalSpeech2.sample`, ns2.py:1496-1499) and
`SEANetEncoder` its `encoder` (24 kHz audio -> 75 Hz frames, what `NaturalSpeech2.forward` and `process_prompt` run on
raw audio).  Each class docstring has its layer table; both are built from the same stages (`_SEANet`), on token-major
activations (B, time, channels), every conv causal with reflect left padding, weight norm folded:
    Conv1d k7                           elu_pad (pad 6) + 7-segment GEMM
    2-layer LSTM(512), lstm(x)[0] + x   input projection GEMM + ns2_lstm_seq per layer
    ResnetBlock(C, hidden C/2), C >= 64 elu_pad (ELU | raw, pad 2) + 3-segment GEMM, elu_pad, one GEMM for
                                        conv1x1 + shortcut over [ELU(x) | x | ELU(h)]
    ConvTranspose1d / Conv1d k 2s stride s      2-segment GEMM (`pack_conv_transpose`, `pack_strided_conv`)
    the 32-channel stage at 24 kHz      one fp32 kernel: ns2_seanet_tail (decoder), ns2_seanet_head (encoder)
GEMM operands are bf16 with fp32 accumulation; activations between layers, the LSTM cell state and the 32-channel
kernels stay fp32.  The state_dicts have the keys and shapes of transformers' `EncodecDecoder` / `EncodecEncoder`;
`load_encodec_state_dict` takes Meta `encodec` (and audiolm's `EncodecWrapper.model`) keys.  Inference only: there is
no backward.
"""
from __future__ import annotations

import re
from collections import OrderedDict
from typing import Dict, Sequence

import torch
from torch import nn

from . import _lib, ops
from .model import _PackedCache

RATIOS = (8, 5, 4, 2)

# the 24 kHz Encodec model's SEANet configuration (transformers EncodecConfig() defaults); nothing else is built
SUPPORTED = dict(audio_channels=1, num_filters=32, upsampling_ratios=(8, 5, 4, 2), hidden_size=128, kernel_size=7,
                 last_kernel_size=7, residual_kernel_size=3, dilation_growth_rate=2, num_residual_layers=1,
                 compress=2, num_lstm_layers=2, use_causal_conv=True, pad_mode="reflect", norm_type="weight_norm",
                 trim_right_ratio=1.0, use_conv_shortcut=True)


# The shortest waveform, in frames, that the encoder reads as a prefix of a longer one.  Every conv pads on the left by
# reflection, and Encodec reflects an input no longer than the pad around appended zeros instead.  The binding stage is
# the last conv (k7, pad 6) at the frame rate: n frames need n > 6.  The others pad at most 8 rows at 8 or more rows
# per frame (pads 6, 2, 2 at 320; 2, 4 at 160; 2, 5 at 40; 2, 8 at 8), so n >= 2 satisfies them.
MIN_FRAMES = 7


def frame_lengths(lengths, batch: int, frames: int, *, device, lo: int = MIN_FRAMES) -> list:
    """Per-sample frame counts of a batch padded at the end, checked before anything runs: one integer per sample (a
    sequence, or an integer tensor on the CPU or on `device`), each in [lo, frames], at most
    NS2_GEMM_ROW_LENS_MAX_BATCHES samples.  Returns them as a list of ints."""
    if isinstance(lengths, torch.Tensor):
        if lengths.is_floating_point() or lengths.is_complex() or lengths.dtype == torch.bool:
            raise ValueError(f"lengths must hold integers, got {lengths.dtype}")
        if lengths.device.type != "cpu" and lengths.device != torch.device(device):
            raise ValueError(f"lengths must be on the CPU or on the audio's device {device}, got {lengths.device}")
        if lengths.dim() > 1:
            raise ValueError(f"lengths must be one-dimensional, got shape {tuple(lengths.shape)}")
        host = [int(v) for v in lengths.tolist()] if lengths.dim() == 1 else [int(lengths)]
    else:
        host = [int(v) for v in lengths]
    if len(host) != batch:
        raise ValueError(f"lengths must hold one length per sample ({batch}), got {len(host)}")
    cap = _lib.NS2_GEMM_ROW_LENS_MAX_BATCHES
    if batch > cap:
        raise ValueError(f"lengths: at most {cap} samples per call, got {batch}")
    if host and min(host) < lo:
        why = " (shorter waveforms fall under Encodec's short-input padding rule when encoded alone)" \
            if lo == MIN_FRAMES else ""
        raise ValueError(f"lengths must be >= {lo} frames{why}, got {min(host)}")
    if host and max(host) > frames:
        raise ValueError(f"the input holds {frames} frames, fewer than the longest length {max(host)} "
                         f"(lengths count frames of 320 samples)")
    return host


def lstm_gate_perm() -> torch.Tensor:
    """Row order of the packed LSTM weights (include/ns2_b200.h section 10): packed row 128 c + 64 hf + 16 w + 8 i + q
    is PyTorch row (2 hf + i) * 512 + 32 c + 8 w + q (gate 2 hf + i of hidden unit 32 c + 8 w + q)."""
    c, hf, w, i, q = torch.meshgrid(*(torch.arange(n) for n in (16, 2, 4, 2, 8)), indexing="ij")
    return ((2 * hf + i) * 512 + 32 * c + 8 * w + q).reshape(-1)


def fold_weight_norm(g: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """w = g v / ||v||, the norm over every dim but 0 (output channels of a Conv1d, input channels of a
    ConvTranspose1d) - torch.nn.utils.parametrizations.weight_norm(dim=0)."""
    return g * v / v.norm(dim=tuple(range(1, v.dim())), keepdim=True)


def pack_conv_transpose(w: torch.Tensor, b: torch.Tensor, s: int):
    """ConvTranspose1d(k = 2s, stride s) weight (C_in, C_out, 2s) and bias -> the 2-segment GEMM's bf16 pack
    (s C_out, 2 C_in) and f32 bias: packed row r C_out + co, column j C_in + ci = w[ci, co, j s + r], so output frame
    n, columns [r C_out, (r + 1) C_out) is output sample s n + r (segment j reads input frame n - j)."""
    c_in, c_out = w.shape[0], w.shape[1]
    packed = w.reshape(c_in, c_out, 2, s).permute(3, 1, 2, 0).reshape(s * c_out, 2 * c_in)
    return packed.to(torch.bfloat16).contiguous(), b.float().repeat(s).contiguous()


def _pack_block32(w3, b3, w1, b1, w_sc, b_sc) -> torch.Tensor:
    """Folded weights of the 32-channel ResnetBlock (conv3 (16, 32, 3), conv1x1 (32, 16, 1), shortcut (32, 32, 1)) ->
    the 3120 floats both full-rate kernels read: w3 (tap, in, out) | b3 | shortcut (in, out) | conv1x1 (in, out) |
    b_sc + b1."""
    return torch.cat([w3.permute(2, 1, 0).reshape(-1), b3, w_sc[:, :, 0].t().reshape(-1), w1[:, :, 0].t().reshape(-1),
                      b_sc + b1])


def pack_tail(w3, b3, w1, b1, w_sc, b_sc, w_f, b_f) -> torch.Tensor:
    """Folded weights of the 32-channel ResnetBlock (`_pack_block32`) and of the final conv (1, 32, 7) -> the
    NS2_SEANET_TAIL_PARAMS f32 layout of ns2_seanet_tail."""
    p = torch.cat([_pack_block32(w3, b3, w1, b1, w_sc, b_sc), w_f[0].t().reshape(-1), b_f.reshape(1),
                   b_f.new_zeros(3)])
    assert p.numel() == _lib.NS2_SEANET_TAIL_PARAMS
    return p.float().contiguous()


def pack_head(w0, b0, w3, b3, w1, b1, w_sc, b_sc) -> torch.Tensor:
    """Folded weights of the encoder's first conv (32, 1, 7) and of its 32-channel ResnetBlock (`_pack_block32`) -> the
    NS2_SEANET_HEAD_PARAMS f32 layout of ns2_seanet_head."""
    p = torch.cat([w0[:, 0].t().reshape(-1), b0, _pack_block32(w3, b3, w1, b1, w_sc, b_sc)])
    assert p.numel() == _lib.NS2_SEANET_HEAD_PARAMS
    return p.float().contiguous()


def _pack_conv(w: torch.Tensor) -> torch.Tensor:
    """Conv1d weight (C_out, C_in, k) -> the k-segment GEMM's bf16 pack (C_out, k C_in), tap-major: column
    j C_in + ci = w[co, ci, j]."""
    return w.permute(0, 2, 1).reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()


def pack_strided_conv(w: torch.Tensor) -> torch.Tensor:
    """Conv1d(k = 2s, stride s) weight (C_out, C_in, 2s) -> the 2-segment GEMM's bf16 pack (C_out, 2s C_in), tap-major:
    column j C_in + ci = w[co, ci, j].  With the input reflect-padded by s and viewed as rows of s samples, segment 0
    (taps [0, s)) reads row m - 1 and segment 1 (taps [s, 2s)) row m: output row m + 1 is conv output m."""
    return _pack_conv(w)


def strided_conv_segs(s: int, c_in: int) -> list:
    """`ns2_gemm` segments of `pack_strided_conv` (include/ns2_b200.h section 10)."""
    return [(0, 0, s * c_in, 1, 0), (0, s * c_in, s * c_in, 0, 0)]


def _check_config(cls_name: str, given: dict) -> None:
    bad = {k: v for k, v in given.items() if v != SUPPORTED[k]}
    if bad:
        raise ValueError(f"{cls_name} supports only the 24 kHz Encodec configuration; unsupported: {bad} "
                         f"(expected {({k: SUPPORTED[k] for k in bad})})")


def encodec_keys_to_transformers(sd: Dict[str, torch.Tensor], part: str) -> Dict[str, torch.Tensor]:
    """Meta `encodec` SEANet keys (`{part}.model.{i}.conv.conv.weight_g|weight_v|bias`, `model.{i}.convtr.convtr.*`,
    `model.{i}.block.{j}.conv.conv.*`, `model.{i}.shortcut.conv.conv.*`, `model.{i}.lstm.*`; the `{part}.` prefix,
    "encoder" or "decoder", is optional) -> transformers' `Encodec{Encoder,Decoder}` keys (`layers.{i}...`)."""
    out = {}
    for k, v in sd.items():
        k = k[len(part) + 1:] if k.startswith(part + ".") else k
        m = re.fullmatch(r"model\.(\d+)\.(.*)", k)
        if m is None:
            raise KeyError(f"unexpected key {k!r} in an encodec {part} state_dict")
        i, rest = m.group(1), m.group(2)
        rest = re.sub(r"^(conv\.conv|convtr\.convtr)\.", "conv.", rest)
        rest = re.sub(r"^(block\.\d+|shortcut)\.conv\.conv\.", r"\1.conv.", rest)
        rest = re.sub(r"conv\.weight_g$", "conv.parametrizations.weight.original0", rest)
        rest = re.sub(r"conv\.weight_v$", "conv.parametrizations.weight.original1", rest)
        out[f"layers.{i}.{rest}"] = v
    return out


class _WNConv(nn.Module):
    """Parameter holder of EncodecConv1d / EncodecConvTranspose1d: `conv` is the weight-normed torch module."""

    def __init__(self, c_in: int, c_out: int, kernel: int, stride: int = 1, transposed: bool = False):
        super().__init__()
        conv = nn.ConvTranspose1d(c_in, c_out, kernel, stride) if transposed else nn.Conv1d(c_in, c_out, kernel, stride)
        self.conv = nn.utils.parametrizations.weight_norm(conv)

    def folded(self):
        p = self.conv.parametrizations.weight
        return fold_weight_norm(p.original0.float(), p.original1.float()), self.conv.bias.float()


class _LSTMParams(nn.Module):
    """Parameter holder of EncodecLSTM."""

    def __init__(self, dim: int, layers: int):
        super().__init__()
        self.lstm = nn.LSTM(dim, dim, layers)


class _ResnetParams(nn.Module):
    """Parameter holder of EncodecResnetBlock: block = [ELU, conv k3 dim -> hidden, ELU, conv k1 hidden -> dim]."""

    def __init__(self, dim: int, hidden: int, kernel: int):
        super().__init__()
        self.block = nn.ModuleList([nn.ELU(), _WNConv(dim, hidden, kernel), nn.ELU(), _WNConv(hidden, dim, 1)])
        self.shortcut = _WNConv(dim, dim, 1)


class _SEANet(_PackedCache):
    """What the two directions share: the constructor's configuration check, the per-shape workspace cache, and the
    packing, workspace buffers and launches of the LSTM and ResnetBlock stages.  A subclass builds its `layers` (the
    only registered sub-module, so the state_dict has transformers' keys), packs them, and runs them."""

    _part: str  # "decoder" or "encoder": the sub-module of Meta's EncodecModel this class loads

    def __init__(self, *, audio_channels: int = 1, num_filters: int = 32, upsampling_ratios: Sequence[int] = RATIOS,
                 hidden_size: int = 128, kernel_size: int = 7, last_kernel_size: int = 7, residual_kernel_size: int = 3,
                 dilation_growth_rate: int = 2, num_residual_layers: int = 1, compress: int = 2,
                 num_lstm_layers: int = 2, use_causal_conv: bool = True, pad_mode: str = "reflect",
                 norm_type: str = "weight_norm", trim_right_ratio: float = 1.0, use_conv_shortcut: bool = True):
        super().__init__()
        given = dict(audio_channels=audio_channels, num_filters=num_filters,
                     upsampling_ratios=tuple(int(r) for r in upsampling_ratios), hidden_size=hidden_size,
                     kernel_size=kernel_size, last_kernel_size=last_kernel_size,
                     residual_kernel_size=residual_kernel_size, dilation_growth_rate=dilation_growth_rate,
                     num_residual_layers=num_residual_layers, compress=compress, num_lstm_layers=num_lstm_layers,
                     use_causal_conv=bool(use_causal_conv), pad_mode=pad_mode, norm_type=norm_type,
                     trim_right_ratio=float(trim_right_ratio), use_conv_shortcut=bool(use_conv_shortcut))
        _check_config(type(self).__name__, given)
        self.layers = nn.ModuleList(self._build_layers(given))
        self._ws: "OrderedDict[tuple, Dict[str, torch.Tensor]]" = OrderedDict()
        # LRU bound on per-shape workspaces: ~10 GB each for the decoder at (B, N) = (32, 1024), ~6.5 GB each for the
        # encoder at (B, T) = (32, 327680)
        self.max_cached_shapes = 4

    @classmethod
    def from_config(cls, config):
        """From an object with transformers' `EncodecConfig` attribute names."""
        return cls(**{k: getattr(config, k) for k in SUPPORTED})

    def load_encodec_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """Load the state_dict of this direction's Meta `encodec` SEANet module (`EncodecModel.decoder` / `.encoder`,
        also audiolm's `EncodecWrapper.model.decoder` / `.encoder`): `model.{i}.conv.conv.weight_g|weight_v|bias`,
        `model.{i}.convtr.convtr.*`, `model.{i}.block.{j}.conv.conv.*`, `model.{i}.shortcut.conv.conv.*`,
        `model.{i}.lstm.*`.  A `decoder.` / `encoder.` prefix is stripped.  The mapping follows the upstream module
        layout; it has not been checked against a released checkpoint, so load with strict=True and compare the output
        for one clip against the original module once."""
        return self.load_state_dict(encodec_keys_to_transformers(sd, self._part), strict=strict)

    @property
    def device(self):
        return next(self.parameters()).device

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._ws.clear()
        return out

    # ----------------------------------------------------------------------------------------------
    # weight packing (folded weight norm, bf16, K-major; rebuilt when a parameter changes)
    # ----------------------------------------------------------------------------------------------
    @staticmethod
    def _pack_lstm(P: Dict[str, torch.Tensor], lstm: nn.LSTM) -> None:
        perm = lstm_gate_perm().to(lstm.weight_ih_l0.device)
        for l in range(2):
            P[f"l{l}_wih"] = getattr(lstm, f"weight_ih_l{l}")[perm].to(torch.bfloat16).contiguous()
            P[f"l{l}_whh"] = getattr(lstm, f"weight_hh_l{l}")[perm].to(torch.bfloat16).contiguous()
            P[f"l{l}_b"] = (getattr(lstm, f"bias_ih_l{l}") + getattr(lstm, f"bias_hh_l{l}"))[perm].float().contiguous()

    @staticmethod
    def _pack_resblock(P: Dict[str, torch.Tensor], si: int, blk: "_ResnetParams") -> None:
        w3, b3 = blk.block[1].folded()                              # (H, D, 3)
        w1, b1 = blk.block[3].folded()                              # (D, H, 1)
        ws, bs = blk.shortcut.folded()                              # (D, D, 1)
        P[f"r{si}_w3"], P[f"r{si}_b3"] = _pack_conv(w3), b3.float().contiguous()
        P[f"r{si}_w1"] = torch.cat([ws[:, :, 0], w1[:, :, 0]], dim=1).to(torch.bfloat16).contiguous()
        P[f"r{si}_b1"] = (bs + b1).float().contiguous()

    # ----------------------------------------------------------------------------------------------
    # workspaces (per input shape, LRU-bounded)
    # ----------------------------------------------------------------------------------------------
    def _workspace(self, B: int, n: int, dev) -> Dict[str, torch.Tensor]:
        key = (B, n, str(dev))
        ws = self._ws.get(key)
        if ws is not None:
            self._ws.move_to_end(key)
            return ws
        while len(self._ws) >= self.max_cached_shapes:
            self._ws.popitem(last=False)
        ws = self._ws[key] = self._alloc_workspace(
            B, n, lambda *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt))
        return ws

    @staticmethod
    def _resblock_ws(ws: Dict[str, torch.Tensor], e, si: int, B: int, L: int, c: int) -> None:
        ws[f"blk{si}"] = e(B, L + 2, 2 * c + c // 2)                # [ELU(x) | x | ELU(h)], reflect-padded by 2
        ws[f"h{si}"] = e(B, L + 2, c // 2, dt=torch.float32)
        ws[f"z{si}"] = e(B, L + 2, c, dt=torch.float32)

    # ----------------------------------------------------------------------------------------------
    # stages
    # ----------------------------------------------------------------------------------------------
    @staticmethod
    def _lstm_stage(P, ws, y: torch.Tensor, out: torch.Tensor, row_lens=None) -> None:
        """out = lstm(y)[0] + y, y and out (B, N, 512) fp32.  row_lens (optional): the input projections compute only
        the 128-row tiles that start before them; the recurrence runs over every row (it is causal)."""
        ops.elu_pad(y, ws["xb"], pad=0, elu=False)
        ops.gemm(ws["xb"], P["l0_wih"], ws["xp"], n=2048, epilogue=ops.EPI_F32, bias=P["l0_b"], row_lens=row_lens)
        ops.lstm_seq(ws["xp"], P["l0_whh"], out_bf16=ws["xb"])
        ops.gemm(ws["xb"], P["l1_wih"], ws["xp"], n=2048, epilogue=ops.EPI_F32, bias=P["l1_b"], row_lens=row_lens)
        ops.lstm_seq(ws["xp"], P["l1_whh"], skip=y, out=out)

    @staticmethod
    def _resblock_stage(P, ws, si: int, x: torch.Tensor, c: int, row_lens=None) -> torch.Tensor:
        """ResnetBlock(c, hidden c / 2) of x (B, L, c) fp32 -> (B, L, c) fp32, a view of `z{si}`.  row_lens (optional):
        per-sample row counts of the padded (B, L + 2) buffers, passed to both GEMMs."""
        h = c // 2
        blk, hb, zo = ws[f"blk{si}"], ws[f"h{si}"], ws[f"z{si}"]
        ops.elu_pad(x, blk, pad=2, elu=True, raw=True)              # [ELU(x) | x], reflect-padded by 2
        ops.gemm(blk, P[f"r{si}_w3"], hb, n=h, epilogue=ops.EPI_F32, segs=ops.conv_segs(c, 3, 2), bias=P[f"r{si}_b3"],
                 row_lens=row_lens)
        ops.elu_pad(hb[:, 2:], blk[:, 2:, 2 * c:], pad=0, elu=True)
        ops.gemm(blk, P[f"r{si}_w1"], zo, n=c, epilogue=ops.EPI_F32,
                 segs=[(c, 0, c, 0, 0), (2 * c, c, h, 0, 0)], bias=P[f"r{si}_b1"], row_lens=row_lens)
        return zo[:, 2:]


class SEANetDecoder(_SEANet):
    """Encodec's SEANet decoder (24 kHz model): (B, N, 128) summed codewords -> (B, 1, 320 N) audio, fp32.

    Layers (transformers `EncodecDecoder` indices):
        0       Conv1d k7 128 -> 512                  elu_pad (pad 6) + 7-segment GEMM
        1       2-layer LSTM(512), lstm(x)[0] + x     the LSTM stage
        2-3     ELU, ConvTranspose1d k16 s8 512 -> 256elu_pad + 2-segment GEMM (taps [0, s) shift 0, [s, 2s) shift 1)
        4       ResnetBlock(256, hidden 128)          the ResnetBlock stage
        5-10    the same at 256 -> 128 (k10 s5) and 128 -> 64 (k8 s4)
        11-12   ELU, ConvTranspose1d k4 s2 64 -> 32   elu_pad + 2-segment GEMM
        13-15   ResnetBlock(32, hidden 16), ELU, Conv1d k7 32 -> 1      ns2_seanet_tail (fp32)
    The constructor takes transformers' `EncodecConfig` decoder fields; only the 24 kHz model's values are supported
    (`SEANetDecoder.from_config(EncodecConfig())` or no arguments)."""

    _part = "decoder"

    def _build_layers(self, c: dict) -> list:
        scale, nf = 2 ** len(RATIOS), c["num_filters"]
        layers = [_WNConv(c["hidden_size"], scale * nf, c["kernel_size"]),
                  _LSTMParams(scale * nf, c["num_lstm_layers"])]
        for r in RATIOS:
            dim = scale * nf
            layers += [nn.ELU(), _WNConv(dim, dim // 2, 2 * r, stride=r, transposed=True),
                       _ResnetParams(dim // 2, dim // 2 // c["compress"], c["residual_kernel_size"])]
            scale //= 2
        return layers + [nn.ELU(), _WNConv(nf, c["audio_channels"], c["last_kernel_size"])]

    def _pack(self) -> Dict[str, torch.Tensor]:
        P = {}
        w, b = self.layers[0].folded()                              # (512, 128, 7)
        P["c0_w"], P["c0_b"] = _pack_conv(w), b.float().contiguous()
        self._pack_lstm(P, self.layers[1].lstm)
        for si, s in enumerate(RATIOS):
            P[f"t{si}_w"], P[f"t{si}_b"] = pack_conv_transpose(*self.layers[3 + 3 * si].folded(), s)
            blk = self.layers[4 + 3 * si]
            if si < len(RATIOS) - 1:
                self._pack_resblock(P, si, blk)
            else:
                P["tail"] = pack_tail(*blk.block[1].folded(), *blk.block[3].folded(), *blk.shortcut.folded(),
                                      *self.layers[15].folded())
        return P

    def _alloc_workspace(self, B: int, N: int, e) -> Dict[str, torch.Tensor]:
        f = torch.float32
        ws = {"a0": e(B, N + 6, 128), "y0": e(B, N + 6, 512, dt=f), "xb": e(B, N, 512), "xp": e(B, N, 2048, dt=f),
              "z": e(B, N, 512, dt=f)}
        L = N
        for si, s in enumerate(RATIOS):
            c_in = 512 >> si
            ws[f"at{si}"] = e(B, L, c_in)
            ws[f"u{si}"] = e(B, L, s * c_in // 2, dt=f)
            L *= s
            if si < len(RATIOS) - 1:
                self._resblock_ws(ws, e, si, B, L, c_in // 2)
        return ws

    @torch.no_grad()
    def forward(self, emb: torch.Tensor) -> torch.Tensor:
        """emb (B, N, 128) -> audio (B, 1, 320 N) fp32."""
        if emb.dim() != 3 or emb.shape[-1] != 128:
            raise ValueError(f"SEANetDecoder takes (B, N, 128) latents, got {tuple(emb.shape)}")
        B, N, _ = emb.shape
        dev = emb.device
        out = torch.empty(B, 1, 320 * N, device=dev, dtype=torch.float32)
        if B == 0 or N == 0:
            return out
        with torch.cuda.device(dev):
            P, ws = self.packed(), self._workspace(B, N, dev)
            x = emb.float().contiguous()
            ops.elu_pad(x, ws["a0"], pad=6, elu=False)
            ops.gemm(ws["a0"], P["c0_w"], ws["y0"], n=512, epilogue=ops.EPI_F32, segs=ops.conv_segs(128, 7, 6),
                     bias=P["c0_b"])
            self._lstm_stage(P, ws, ws["y0"][:, 6:], ws["z"])
            z, L = ws["z"], N
            for si, s in enumerate(RATIOS):
                c_in = 512 >> si
                c_out = c_in // 2
                at, u = ws[f"at{si}"], ws[f"u{si}"]
                ops.elu_pad(z, at, pad=0, elu=True)
                ops.gemm(at, P[f"t{si}_w"], u, n=s * c_out, epilogue=ops.EPI_F32,
                         segs=[(0, 0, c_in, 0, 0), (0, c_in, c_in, 1, 0)], bias=P[f"t{si}_b"])
                L *= s
                u = u.view(B, L, c_out)
                if si == len(RATIOS) - 1:
                    ops.seanet_tail(u, P["tail"], out.view(B, L))
                    break
                z = self._resblock_stage(P, ws, si, u, c_out)
        return out


class SEANetEncoder(_SEANet):
    """Encodec's SEANet encoder (24 kHz model): (B, T) or (B, 1, T) audio, T a multiple of 320 -> (B, T / 320, 128)
    token-major frames, fp32 — the `encoder` callable of `EncodecRVQ`.

    Layers (transformers `EncodecEncoder` indices):
        0-2     Conv1d k7 1 -> 32, ResnetBlock(32, hidden 16), ELU      ns2_seanet_head (fp32, bf16 output)
        3       Conv1d k4 stride 2 32 -> 64                             2-segment GEMM (`strided_conv_segs`)
        4-5     ResnetBlock(64, hidden 32), ELU                         the ResnetBlock stage, then elu_pad (pad s)
        6-11    the same at k8 s4 64 -> 128, ResnetBlock(128); k10 s5 128 -> 256, ResnetBlock(256)
        12      Conv1d k16 stride 8 256 -> 512                          2-segment GEMM
        13      2-layer LSTM(512), lstm(x)[0] + x                       the LSTM stage
        14-15   ELU, Conv1d k7 512 -> 128                               elu_pad (pad 6) + 7-segment GEMM, fp32 out
    The constructor takes transformers' `EncodecConfig` fields; only the 24 kHz model's values are supported."""

    _part = "encoder"

    def _build_layers(self, c: dict) -> list:
        dim = c["num_filters"]
        layers = [_WNConv(c["audio_channels"], dim, c["kernel_size"])]
        for r in reversed(RATIOS):
            layers += [_ResnetParams(dim, dim // c["compress"], c["residual_kernel_size"]), nn.ELU(),
                       _WNConv(dim, 2 * dim, 2 * r, stride=r)]
            dim *= 2
        return layers + [_LSTMParams(dim, c["num_lstm_layers"]), nn.ELU(),
                         _WNConv(dim, c["hidden_size"], c["last_kernel_size"])]

    def _pack(self) -> Dict[str, torch.Tensor]:
        P = {}
        blk = self.layers[1]
        P["head"] = pack_head(*self.layers[0].folded(), *blk.block[1].folded(), *blk.block[3].folded(),
                              *blk.shortcut.folded())
        for si in range(len(RATIOS)):
            w, b = self.layers[3 + 3 * si].folded()                 # (2C, C, 2s)
            P[f"s{si}_w"], P[f"s{si}_b"] = pack_strided_conv(w), b.float().contiguous()
            if si < len(RATIOS) - 1:
                self._pack_resblock(P, si, self.layers[4 + 3 * si])
        self._pack_lstm(P, self.layers[13].lstm)
        w, b = self.layers[15].folded()                             # (128, 512, 7)
        P["c15_w"], P["c15_b"] = _pack_conv(w), b.float().contiguous()
        return P

    def _alloc_workspace(self, B: int, T: int, e) -> Dict[str, torch.Tensor]:
        f = torch.float32
        strides = tuple(reversed(RATIOS))
        ws = {"a0": e(B, T + strides[0], 32)}
        L = T
        for si, s in enumerate(strides):
            c_out = 64 << si
            L //= s
            ws[f"y{si}"] = e(B, L + 1, c_out, dt=f)                 # row 0: the strided GEMM's scratch row
            if si < len(strides) - 1:
                self._resblock_ws(ws, e, si, B, L, c_out)
                ws[f"a{si + 1}"] = e(B, L + strides[si + 1], c_out)
        N = L
        ws.update(xb=e(B, N, 512), xp=e(B, N, 2048, dt=f), lz=e(B, N, 512, dt=f), a15=e(B, N + 6, 512))
        return ws

    @torch.no_grad()
    def forward(self, audio: torch.Tensor, *, lengths=None) -> torch.Tensor:
        """audio (B, T) or (B, 1, T), T % 320 == 0 -> frames (B, T / 320, 128) fp32, a new tensor per call.

        lengths (B,) (optional, frames, in [MIN_FRAMES, T / 320], at most NS2_GEMM_ROW_LENS_MAX_BATCHES samples): a
        batch of waveforms padded at the end, sample b being audio[b, :320 lengths[b]].  Its frames [0, lengths[b]) are
        then bit-identical to encoding that waveform alone, whatever the padding holds (NaN included), and its frames
        past it are exact zeros.  Every conv GEMM computes only the 128-row tiles that start before a sample's length
        at its rate; the full-rate head, the operand preparation and the LSTM recurrence run over the padded rows."""
        if audio.dim() == 3 and audio.shape[1] == 1:
            audio = audio[:, 0]
        if audio.dim() != 2:
            raise ValueError(f"SEANetEncoder takes (B, T) or (B, 1, T) audio, got {tuple(audio.shape)}")
        B, T = audio.shape
        if T % 320:
            raise ValueError(f"SEANetEncoder needs T % 320 == 0 (the product of the strides), got T={T}")
        dev = audio.device
        N = T // 320
        host_lens = None if lengths is None else frame_lengths(lengths, B, N, device=dev)
        if B == 0 or T == 0:
            return torch.empty(B, N, 128, device=dev, dtype=torch.float32)
        frames = torch.empty(B, N + 6, 128, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            strides = tuple(reversed(RATIOS))
            rl = {}   # per-stage GEMM row counts: padded buffers hold 1 (strided), 2 (ResnetBlock) or 6 leading rows
            if host_lens is not None:
                def rows(pad, rate, name):
                    return ops.lengths([pad + n * rate for n in host_lens], B, None, device=dev, name=name)
                rate = 320
                for si, s in enumerate(strides):
                    rate //= s
                    rl[f"s{si}"] = rows(1, rate, f"stride {s} conv rows")
                    if si < len(strides) - 1:
                        rl[f"r{si}"] = rows(2, rate, f"ResnetBlock {si} rows")
                rl["lstm"], rl["c15"] = rows(0, 1, "frames"), rows(6, 1, "last conv rows")
            P, ws = self.packed(), self._workspace(B, T, dev)
            x = audio.float()
            if x.stride(1) != 1:
                x = x.contiguous()
            a, L, c_in = ws["a0"], T, 32
            ops.seanet_head(x, P["head"], a)                       # bf16(ELU(z1)) reflect-padded by 2
            for si, s in enumerate(strides):
                c_out = 2 * c_in
                L //= s
                y = ws[f"y{si}"]
                ops.gemm(a.view(B, L + 1, s * c_in), P[f"s{si}_w"], y, n=c_out, epilogue=ops.EPI_F32,
                         segs=strided_conv_segs(s, c_in), bias=P[f"s{si}_b"], row_lens=rl.get(f"s{si}"))
                y = y[:, 1:]
                if si == len(strides) - 1:
                    break
                a = ws[f"a{si + 1}"]
                ops.elu_pad(self._resblock_stage(P, ws, si, y, c_out, row_lens=rl.get(f"r{si}")), a,
                            pad=strides[si + 1], elu=True)
                c_in = c_out
            self._lstm_stage(P, ws, y, ws["lz"], row_lens=rl.get("lstm"))
            ops.elu_pad(ws["lz"], ws["a15"], pad=6, elu=True)
            ops.gemm(ws["a15"], P["c15_w"], frames, n=128, epilogue=ops.EPI_F32, segs=ops.conv_segs(512, 7, 6),
                     bias=P["c15_b"], row_lens=rl.get("c15"))
            if host_lens is not None:
                ops.mask_rows(frames[:, 6:], rl["lstm"])
        return frames[:, 6:]
