"""FACodecDecoder — drop-in for the decoder of NaturalSpeech 3's FACodec (``models/codec/ns3_codec/facodec.py:242``):
the same constructor, the same parameter tree (``quantizer.{q}.layers.{j}.{in_proj,out_proj,_codebook}``, ``model.*``,
``timbre_encoder.*``, ``timbre_linear``, the ``CNNLSTM`` predictors and the ``use_gr_*`` heads), so the released
``ns3_facodec_decoder.bin`` loads strictly.  Served natively (``AB_GEN_FACODEC``):

- ``forward(x, vq=True)`` in eval: latent ``[B, in_channels, T]`` -> ``(outs, qs, commit_loss, quantized_buf,
  spk_embs)`` (:408-471): the three ResidualVQs on fp32 CUDA cores (codes are discrete) and the timbre transformer;
  needs ``in_channels == 256``, the timbre encoder's width;
- ``vq2emb(vq, use_residual_code=True)``: codes ``[n_q, B, T]`` -> ``[B, in_channels, T]`` (:556-566);
- ``inference(x, speaker_embedding)``: the timbre FiLM (LayerNorm over channels, ``x * gamma + beta``) and the
  BigVGAN-family generator -> ``[B, 1, T * prod(up_ratios)]`` (:568-576).

``FACodecEncoder`` (:157-194) serves the waveform -> latent side natively (``AB_GEN_FACODEC_ENCODER``): ``forward`` /
``inference`` map ``[B, 1, N]`` to ``[B, out_channels, F]`` through the same ResidualUnits and strided convolutions.

``FACodecRedecoder`` (:602-769) serves the README's zero-shot voice conversion natively (``AB_GEN_FACODEC_REDECODER``):
``vq2emb(vq, speaker_embedding, use_residual=True)`` gathers the prosody codes' embeddings, runs them through the
speaker-conditioned prosody transformer (style-adaptive LayerNorms) and adds the content and residual embeddings ->
``[B, 256, T]``; ``inference`` is the decoder's.  Its ``forward`` is broken in the reference and is refused.

``FACodecEncoderV2`` / ``FACodecDecoderV2`` (:772-1199) serve the README's second voice-conversion flow: the encoder adds
``get_prosody_feature`` (the first 20 rows of an 80-row log-mel on the native mel pipeline), and the decoder's
``forward(x, prosody_feature, vq=True)`` quantizes the prosody group from ``melspec_encoder(melspec_linear(feature))``,
a second transformer that runs in fp32 at every precision.

The training branch (``vq=False``: the predictors, random residual masking, the losses), ``get_vq`` and a quantizer or
transformer in training mode are not served; the modules only those evaluate are kept as parameters."""
from __future__ import annotations

import numpy as np
import torch
from torch import nn
from torch.nn.utils import remove_weight_norm, weight_norm

from .. import _capi
from .activations import Activation1d, SnakeBeta
from .generator import NativeGenerator

_SERVED = ("amphion_b200 serves FACodecEncoder.forward() / .inference(), FACodecDecoder.forward(vq=True) in eval, "
           "FACodecDecoder.vq2emb() and FACodecDecoder.inference(), and FACodecRedecoder.vq2emb() in eval and "
           "FACodecRedecoder.inference()")
_SERVED_V2 = ("amphion_b200 serves FACodecEncoderV2.forward() / .inference() / .get_prosody_feature(), "
              "FACodecDecoderV2.forward(x, prosody_feature, vq=True) in eval, FACodecDecoderV2.vq2emb() and "
              "FACodecDecoderV2.inference()")


def _native_only(name):
    raise RuntimeError(f"amphion_b200: FACodec's {name} executes inside the decoder's CUDA pipeline; {_SERVED}")


def _act(ch):
    return Activation1d(activation=SnakeBeta(ch, alpha_logscale=True))


class ResidualUnit(nn.Module):
    """Parameter holder for facodec.py:121-133: act, WNConv1d(k = 7, dilation), act, WNConv1d(k = 1)."""

    def __init__(self, dim: int = 16, dilation: int = 1):
        super().__init__()
        pad = ((7 - 1) * dilation) // 2
        self.block = nn.Sequential(
            _act(dim), weight_norm(nn.Conv1d(dim, dim, kernel_size=7, dilation=dilation, padding=pad)),
            _act(dim), weight_norm(nn.Conv1d(dim, dim, kernel_size=1)))

    def forward(self, x):
        _native_only("ResidualUnit")


class DecoderBlock(nn.Module):
    """Parameter holder for facodec.py:220-239."""

    def __init__(self, input_dim: int = 16, output_dim: int = 8, stride: int = 1):
        super().__init__()
        self.block = nn.Sequential(
            _act(input_dim),
            weight_norm(nn.ConvTranspose1d(input_dim, output_dim, kernel_size=2 * stride, stride=stride,
                                           padding=stride // 2 + stride % 2, output_padding=stride % 2)),
            ResidualUnit(output_dim, dilation=1), ResidualUnit(output_dim, dilation=3), ResidualUnit(output_dim, dilation=9))

    def forward(self, x):
        _native_only("DecoderBlock")


class FactorizedVectorQuantize(nn.Module):
    """Parameter holder for quantize/fvq.py:16-29 (dim != codebook_dim: weight-normed in_proj / out_proj)."""

    def __init__(self, dim, codebook_size, codebook_dim, commitment=0.005, **kwargs):
        super().__init__()
        self.codebook_size, self.codebook_dim, self.commitment = codebook_size, codebook_dim, commitment
        self.in_proj = weight_norm(nn.Linear(dim, codebook_dim))
        self.out_proj = weight_norm(nn.Linear(codebook_dim, dim))
        self._codebook = nn.Embedding(codebook_size, codebook_dim)

    def forward(self, *args, **kwargs):
        raise NotImplementedError(f"FACodec quantization is not served; {_SERVED}")


class ResidualVQ(nn.Module):
    """Parameter holder for quantize/rvq.py:12-25."""

    def __init__(self, *, num_quantizers, codebook_size, **kwargs):
        super().__init__()
        if isinstance(codebook_size, int):
            codebook_size = [codebook_size] * num_quantizers
        self.layers = nn.ModuleList([FactorizedVectorQuantize(codebook_size=2 ** s, **kwargs) for s in codebook_size])
        self.num_quantizers = num_quantizers

    def forward(self, *args, **kwargs):
        raise NotImplementedError(f"FACodec quantization is not served; {_SERVED}")


class _Holder(nn.Module):
    def forward(self, *args, **kwargs):
        raise NotImplementedError(f"amphion_b200: {type(self).__name__} is not served; {_SERVED}")


class GradientReversal(_Holder):
    """gradient_reversal.py:29-35 (no state-dict entries)."""

    def __init__(self, alpha):
        super().__init__()
        self.alpha = torch.tensor(alpha, requires_grad=False)


class CNNLSTM(_Holder):
    """Parameter holder for facodec.py:35-54 (the f0 / phone predictors)."""

    def __init__(self, indim, outdim, head, global_pred=False):
        super().__init__()
        self.global_pred = global_pred
        self.model = nn.Sequential(ResidualUnit(indim, dilation=1), ResidualUnit(indim, dilation=2),
                                   ResidualUnit(indim, dilation=3), _act(indim))
        self.heads = nn.ModuleList([nn.Linear(indim, outdim) for _ in range(head)])


class _PositionalEncoding(_Holder):
    """transformer.py:35-47: the persistent ``pe`` buffer [max_len, 1, d_model]."""

    def __init__(self, d_model, max_len=5000):
        super().__init__()
        self.register_buffer("pe", torch.zeros(max_len, 1, d_model))


class _FFN(_Holder):
    def __init__(self, hidden, filt, k):
        super().__init__()
        self.ffn_1 = nn.Conv1d(hidden, filt, k, padding=k // 2)
        self.ffn_2 = nn.Linear(filt, hidden)


class StyleAdaptiveLayerNorm(_Holder):
    """Parameter holder for transformer.py:13-32: ``gamma * LayerNorm(x) + beta`` (no affine, eps 1e-5) with
    ``(gamma, beta) = style(mean(condition, dim=1))``."""

    def __init__(self, normalized_shape):
        super().__init__()
        self.style = nn.Linear(normalized_shape, 2 * normalized_shape)
        self.style.bias.data[:normalized_shape] = 1
        self.style.bias.data[normalized_shape:] = 0


class _EncoderLayer(_Holder):
    def __init__(self, hidden, heads, filt, k, use_cln=False):
        super().__init__()
        norm = StyleAdaptiveLayerNorm if use_cln else nn.LayerNorm
        self.ln_1 = norm(hidden)
        self.ln_2 = norm(hidden)
        self.self_attn = nn.MultiheadAttention(hidden, heads, batch_first=True)
        self.ffn = _FFN(hidden, filt, k)


class TransformerEncoder(_Holder):
    """Parameter holder for transformer.py:154-234: the decoder's timbre encoder (use_cln=False) or the redecoder's
    speaker-conditioned prosody encoder (use_cln=True: style-adaptive ln_1, ln_2 and last_ln)."""

    def __init__(self, encoder_layer=4, encoder_hidden=256, encoder_head=4, conv_filter_size=1024, conv_kernel_size=5,
                 use_cln=False):
        super().__init__()
        self.position_emb = _PositionalEncoding(encoder_hidden)
        self.layers = nn.ModuleList([_EncoderLayer(encoder_hidden, encoder_head, conv_filter_size, conv_kernel_size,
                                                   use_cln) for _ in range(encoder_layer)])
        self.last_ln = StyleAdaptiveLayerNorm(encoder_hidden) if use_cln else nn.LayerNorm(encoder_hidden)


def _block_config(kind, n_in, channels, up_ratios):
    """The fixed fields of every FACodec generator: a stage per ratio u (kernel 2u), one ResidualUnit kernel (k = 7,
    dilations 1, 3, 9) and SnakeBeta with logscale."""
    c = _capi.GeneratorConfig()
    c.kind, c.n_mel, c.upsample_initial_channel = kind, n_in, channels
    c.num_upsamples = len(up_ratios)
    for i, u in enumerate(up_ratios):
        c.upsample_rates[i], c.upsample_kernel_sizes[i] = u, 2 * u
    c.resblock, c.num_kernels, c.resblock_kernel_sizes[0], c.num_dilations[0] = 1, 1, 7, 3
    for p, d in enumerate((1, 3, 9)):
        c.resblock_dilation_sizes[0][p] = d
    c.activation, c.snake_logscale = _capi.ACT_SNAKEBETA, 1
    return c


def _generator_config(m, kind):
    """The BigVGAN-family generator fields of the decoder and the redecoder (model.*, facodec.py:220-240)."""
    if len(m.up_ratios) > _capi.AB_MAX_STAGES:
        raise ValueError(f"amphion_b200: too many up_ratios for the native {type(m).__name__}")
    c = _block_config(kind, m.in_channels, m.upsample_initial_channel, m.up_ratios)
    for i, (n, bits) in enumerate(((m.vq_num_q_p, m.codebook_size_prosody), (m.vq_num_q_c, m.codebook_size_content),
                                   (m.vq_num_q_r, m.codebook_size_residual))):
        c.vq_num_q[i], c.vq_codebook_bits[i] = n, int(bits)
    return c


def _build_generator(m, in_channels, upsample_initial_channel, up_ratios, timbre_encoder=False):
    """The decoder's and the redecoder's ``model.*``, ``timbre_linear`` and ``timbre_norm`` (facodec.py:337-369,
    :656-677); with ``timbre_encoder``, the decoder's timbre encoder between them.  The order is the reference's, so a
    seeded construction draws the same initial weights."""
    channels = upsample_initial_channel
    layers = [weight_norm(nn.Conv1d(in_channels, channels, kernel_size=7, padding=3))]
    for i, stride in enumerate(up_ratios):
        layers.append(DecoderBlock(channels // 2 ** i, channels // 2 ** (i + 1), stride))
    output_dim = channels // 2 ** len(up_ratios)
    layers += [_act(output_dim), weight_norm(nn.Conv1d(output_dim, 1, kernel_size=7, padding=3)), nn.Tanh()]
    m.model = nn.Sequential(*layers)
    if timbre_encoder:
        m.timbre_encoder = TransformerEncoder()
    m.timbre_linear = nn.Linear(in_channels, in_channels * 2)
    m.timbre_linear.bias.data[:in_channels] = 1
    m.timbre_linear.bias.data[in_channels:] = 0
    m.timbre_norm = nn.LayerNorm(in_channels, elementwise_affine=False)


def _refuse_training(module, what, why, served):
    """Dropout and the training losses are not served: refuse ``module`` when it or a submodule is in training mode."""
    if any(m.training for m in module.modules()):
        raise NotImplementedError(f"amphion_b200: {what} in training mode ({why}) is not served; {served}")


def _check_codes(m, vq, use_residual, who, table):
    """Codes the kernel would not read (it writes NaN there): refuse them before the launch, as F.embedding does."""
    p, c, r = m.vq_num_q_p, m.vq_num_q_c, m.vq_num_q_r
    groups = [(0, p, m.codebook_size_prosody), (p, p + c, m.codebook_size_content)]
    if use_residual and r > 0:
        groups.append((p + c, p + c + r, m.codebook_size_residual))
    for q0, q1, bits in groups:
        part = vq[q0:q1]
        lo, hi = int(part.min()), int(part.max())
        if lo < 0 or hi >= 2 ** int(bits):
            raise ValueError(f"{who}.vq2emb: code rows {q0}..{q1 - 1} hold {lo}..{hi}, outside the {table} "
                             f"[0, {2 ** int(bits)})")


class _FACodecGenerator(NativeGenerator):
    """The hooks the FACodec encoder, decoder and redecoder share."""

    def _input_channels(self):
        return self.in_channels

    def _hop(self):
        return self.hop_length

    def _upsample_rates(self):
        return list(self.up_ratios)

    def remove_weight_norm(self):
        def _remove(mod):
            try:
                remove_weight_norm(mod)
            except ValueError:   # this module has no weight norm
                return
        self.apply(_remove)
        self.invalidate()


def _inference(m, x, speaker_embedding, out, tail_events):
    """FACodecDecoder.inference / FACodecRedecoder.inference (facodec.py:568-576, :761-769) on the native handle."""
    who = type(m).__name__
    if x.dim() != 3 or x.shape[1] != m.in_channels:
        raise ValueError(f"{who}.inference expects x of shape [B, {m.in_channels}, T], got {tuple(x.shape)}")
    spk = speaker_embedding
    if spk.dim() != 2 or spk.shape[1] != m.in_channels or spk.shape[0] != x.shape[0]:
        raise ValueError(f"{who}.inference expects a speaker embedding of shape [{x.shape[0]}, "
                         f"{m.in_channels}], got {tuple(spk.shape)}")
    if spk.device != x.device:
        raise ValueError(f"{who}.inference: x and the speaker embedding are on different devices")
    B, _, T = x.shape
    if B == 0 or T == 0:
        raise ValueError("amphion_b200: empty latent batch")
    _capi.require_cuda(x, f"{who}.inference")
    if x.dtype != torch.float32:
        x = x.float()
    spk = spk.float()
    if spk.stride(1) != 1:
        spk = spk.contiguous()
    with m._launch(x.device) as h:
        need = _capi.lib.ab_generator_workspace_bytes(h, B, T)
        ws = m._scratch(need, x.device)
        wav = m._output(out, (B, 1, T * m.hop_length), x.device)
        m._arm_tail_events(tail_events)
        _capi.check(_capi.lib.ab_facodec_inference(h, _capi.ptr(x), B, T, _capi.shape_array(x.stride()),
                                                   _capi.ptr(spk), spk.stride(0), _capi.ptr(wav), ws, need,
                                                   _capi.stream_ptr()), "ab_facodec_inference")
    return wav


class FACodecDecoder(_FACodecGenerator):
    kind = "facodec"

    def __init__(self, in_channels=256, upsample_initial_channel=1536, ngf=32, up_ratios=(5, 5, 4, 2), vq_num_q_c=2,
                 vq_num_q_p=1, vq_num_q_r=3, vq_dim=1024, vq_commit_weight=0.005, vq_weight_init=False,
                 vq_full_commit_loss=False, codebook_dim=8, codebook_size_prosody=10, codebook_size_content=10,
                 codebook_size_residual=10, quantizer_dropout=0.0, dropout_type="linear", use_gr_content_f0=False,
                 use_gr_prosody_phone=False, use_gr_residual_f0=False, use_gr_residual_phone=False,
                 use_gr_x_timbre=False, use_random_mask_residual=True, prob_random_mask_residual=0.75):
        super().__init__()
        if in_channels != vq_dim:
            # vq2emb's output is inference's input (README flow): the two widths must agree
            raise ValueError(f"amphion_b200: FACodecDecoder needs in_channels == vq_dim (got {in_channels}, {vq_dim})")
        if codebook_dim == vq_dim:
            raise ValueError("amphion_b200: FACodecDecoder with codebook_dim == vq_dim (identity projections) is not served")
        self.hop_length = int(np.prod(up_ratios))
        self.ngf = ngf
        self.up_ratios = [int(u) for u in up_ratios]
        self.in_channels, self.upsample_initial_channel = int(in_channels), int(upsample_initial_channel)
        self.use_random_mask_residual = use_random_mask_residual
        self.prob_random_mask_residual = prob_random_mask_residual
        self.vq_num_q_p, self.vq_num_q_c, self.vq_num_q_r = int(vq_num_q_p), int(vq_num_q_c), int(vq_num_q_r)
        self.codebook_size_prosody = codebook_size_prosody
        self.codebook_size_content = codebook_size_content
        self.codebook_size_residual = codebook_size_residual
        self.codebook_dim = int(codebook_dim)
        # set by the first forward(vq=True): the native handle then also holds the quantizers' in_proj and the timbre
        # encoder (a decode-only handle keeps exactly the decoder's tensors)
        self._quantize_handle = False

        def rvq(n, size):
            return ResidualVQ(num_quantizers=n, dim=vq_dim, codebook_size=size, codebook_dim=codebook_dim,
                              commitment=vq_commit_weight)

        self.quantizer = nn.ModuleList([rvq(vq_num_q_p, codebook_size_prosody), rvq(vq_num_q_c, codebook_size_content)])
        if self.vq_num_q_r > 0:
            self.quantizer.append(rvq(vq_num_q_r, codebook_size_residual))

        _build_generator(self, in_channels, upsample_initial_channel, up_ratios, timbre_encoder=True)
        self.f0_predictor = CNNLSTM(in_channels, 1, 2)
        self.phone_predictor = CNNLSTM(in_channels, 5003, 1)
        self.use_gr_content_f0 = use_gr_content_f0
        self.use_gr_prosody_phone = use_gr_prosody_phone
        self.use_gr_residual_f0 = use_gr_residual_f0
        self.use_gr_residual_phone = use_gr_residual_phone
        self.use_gr_x_timbre = use_gr_x_timbre
        if self.vq_num_q_r > 0 and use_gr_residual_f0:
            self.res_f0_predictor = nn.Sequential(GradientReversal(alpha=1.0), CNNLSTM(in_channels, 1, 2))
        if self.vq_num_q_r > 0 and use_gr_residual_phone > 0:
            self.res_phone_predictor = nn.Sequential(GradientReversal(alpha=1.0), CNNLSTM(in_channels, 5003, 1))
        if use_gr_content_f0:
            self.content_f0_predictor = nn.Sequential(GradientReversal(alpha=1.0), CNNLSTM(in_channels, 1, 2))
        if use_gr_prosody_phone:
            self.prosody_phone_predictor = nn.Sequential(GradientReversal(alpha=1.0), CNNLSTM(in_channels, 5003, 1))
        if use_gr_x_timbre:
            self.x_timbre_predictor = nn.Sequential(GradientReversal(alpha=1),
                                                    CNNLSTM(in_channels, 245200, 1, global_pred=True))

    # ---- NativeGenerator hooks -------------------------------------------------------
    def _c_config_decode(self):
        c = _generator_config(self, _capi.GEN_FACODEC)
        c.vq_codebook_dim = self.codebook_dim
        return c

    def _c_config(self):
        c = self._c_config_decode()
        c.facodec_quantize = int(self._quantize_handle)
        return c

    # ---- served methods --------------------------------------------------------------
    def vq2emb(self, vq, use_residual_code=True):
        """codes [n_q, B, T] (integer, any strides) -> [B, in_channels, T] fp32 on the codes' device."""
        n_pc = self.vq_num_q_p + self.vq_num_q_c
        n_all = n_pc + self.vq_num_q_r
        if vq.dim() != 3 or vq.is_floating_point() or vq.is_complex():
            raise ValueError(f"FACodecDecoder.vq2emb expects integer codes [n_q, B, T], got {vq.dtype} {tuple(vq.shape)}")
        n_q, B, T = vq.shape
        if n_q != n_all and not (not use_residual_code and n_q == n_pc):
            raise ValueError(f"FACodecDecoder.vq2emb: {n_q} code rows, the decoder has {n_all} "
                             f"({self.vq_num_q_p} prosody, {self.vq_num_q_c} content, {self.vq_num_q_r} residual)")
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty code batch")
        _capi.require_cuda(vq, "FACodecDecoder.vq2emb")
        vq = vq.long()
        _check_codes(self, vq, use_residual_code, "FACodecDecoder", "codebook")
        with self._launch(vq.device) as h:
            out = torch.empty(B, self.in_channels, T, dtype=torch.float32, device=vq.device)
            _capi.check(_capi.lib.ab_facodec_vq2emb(h, _capi.ptr(vq), _capi.shape_array(vq.stride()), n_q, B, T,
                                                    int(bool(use_residual_code)), _capi.ptr(out), _capi.stream_ptr()),
                        "ab_facodec_vq2emb")
        return out

    def inference(self, x, speaker_embedding, out=None, tail_events=None):
        """x [B, in_channels, T] (any strides), speaker_embedding [B, in_channels] -> wav [B, 1, T * hop] fp32.

        ``out`` / ``tail_events`` (beyond the reference signature) behave as in the other generators' forward."""
        return _inference(self, x, speaker_embedding, out, tail_events)

    def forward(self, x=None, vq=True, get_vq=False, eval_vq=True, speaker_embedding=None, n_quantizers=None,
                quantized=None):
        """``vq=True``: x [B, 256, T] fp32 (any strides) -> ``(outs [B, 256, T], qs int64 [n_used, B, T],
        commit_loss zeros [n_used], quantized_buf [2 or 3 x [B, 256, T]], spk_embs [B, 256])`` on x's device, without
        autograd history (facodec.py:448-471 in eval).  ``n_quantizers = k`` keeps the first k layers of each group."""
        if get_vq:
            raise NotImplementedError(f"amphion_b200: FACodecDecoder.forward(get_vq=True) is not served; {_SERVED}")
        if vq is not True:
            raise NotImplementedError(f"amphion_b200: the training branch of FACodecDecoder.forward (the predictors, "
                                      f"random residual masking) is not served; {_SERVED}")
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            dev = x.device if isinstance(x, torch.Tensor) else type(x).__name__
            raise NotImplementedError(f"amphion_b200: FACodecDecoder.forward(vq=True) needs a CUDA tensor (got "
                                      f"'{dev}'); there is no CPU fallback; {_SERVED}")
        if self.in_channels != 256:
            raise ValueError(f"amphion_b200: FACodecDecoder.forward(vq=True) needs in_channels == 256, the timbre "
                             f"encoder's width (got {self.in_channels})")
        if x.dim() != 3 or x.shape[1] != self.in_channels:
            raise ValueError(f"FACodecDecoder.forward expects x of shape [B, {self.in_channels}, T], got {tuple(x.shape)}")
        B, _, T = x.shape
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty latent batch")
        return self._quantize(x, None, n_quantizers, eval_vq)

    def _quantize(self, x, pf, n_quantizers, eval_vq):
        """forward(vq=True) once its arguments are checked: V1 (``pf`` None) quantizes the prosody group from x, V2 from
        ``pf``, the prosody feature, through the melspec encoder."""
        served = _SERVED if pf is None else _SERVED_V2
        # the transformers the pass runs, under the names the refusals give them
        encoders = {"timbre encoder": self.timbre_encoder} if pf is None else \
            {"timbre_encoder": self.timbre_encoder, "melspec_encoder": self.melspec_encoder}
        B, _, T = x.shape
        n_pe = min(e.position_emb.pe.shape[0] for e in encoders.values())
        if B > n_pe:
            rows = "the timbre encoder's" if pf is None else "the transformers'"
            raise ValueError(f"amphion_b200: batch {B} > {n_pe}, the rows of {rows} positional encoding (the reference "
                             f"fails there too)")
        k = max(self.vq_num_q_p, self.vq_num_q_c, self.vq_num_q_r) if n_quantizers is None else int(n_quantizers)
        if k < 1:
            raise ValueError(f"amphion_b200: n_quantizers {n_quantizers} < 1 runs no layer (the reference raises too)")
        if eval_vq:
            self.quantizer.eval()   # facodec.py:460-461, :1076-1077
        _refuse_training(self.quantizer, "a quantizer", "quantizer dropout, commitment losses", served)
        for name, mod in encoders.items():
            _refuse_training(mod, f"the {name}", "dropout", served)
        if not self._quantize_handle:
            # the decode-only handle lists no quantizer / transformer tensors: re-create it with them
            self._quantize_handle = True
            if self._handle is not None:
                _capi.lib.ab_generator_destroy(self._handle)
                self._handle = None
            self._arena_key = None
        x = x.float()
        nq = [min(k, n) for n in (self.vq_num_q_p, self.vq_num_q_c, self.vq_num_q_r)]
        n_used, G = sum(nq), 3 if self.vq_num_q_r > 0 else 2
        dev = x.device
        with self._launch(dev) as h:
            need = _capi.lib.ab_facodec_quantize_workspace_bytes(h, B, T)
            ws = self._scratch(need, dev)
            outs = torch.empty(B, self.in_channels, T, dtype=torch.float32, device=dev)
            qs = torch.empty(n_used, B, T, dtype=torch.int64, device=dev)
            buf = torch.empty(G, B, self.in_channels, T, dtype=torch.float32, device=dev)
            spk = torch.empty(B, self.in_channels, dtype=torch.float32, device=dev)
            xs = _capi.shape_array(x.stride())
            if pf is None:
                _capi.check(_capi.lib.ab_facodec_quantize(h, _capi.ptr(x), xs, B, T, k, _capi.ptr(outs), _capi.ptr(qs),
                                                          _capi.ptr(buf), _capi.ptr(spk), ws, need, _capi.stream_ptr()),
                            "ab_facodec_quantize")
            else:
                pf = pf.float()
                _capi.check(_capi.lib.ab_facodec_quantize_prosody(h, _capi.ptr(x), xs, _capi.ptr(pf),
                                                                  _capi.shape_array(pf.stride()), B, T, k,
                                                                  _capi.ptr(outs), _capi.ptr(qs), _capi.ptr(buf),
                                                                  _capi.ptr(spk), ws, need, _capi.stream_ptr()),
                            "ab_facodec_quantize_prosody")
        commit_loss = torch.zeros(n_used, dtype=torch.float32, device=dev)
        return outs, qs, commit_loss, list(buf.unbind(0)), spk


class EncoderBlock(nn.Module):
    """Parameter holder for facodec.py:136-154: three ResidualUnits at dim // 2, act, WNConv1d(dim // 2, dim, k = 2s,
    stride s, padding s//2 + s%2)."""

    def __init__(self, dim: int = 16, stride: int = 1):
        super().__init__()
        self.block = nn.Sequential(
            ResidualUnit(dim // 2, dilation=1), ResidualUnit(dim // 2, dilation=3), ResidualUnit(dim // 2, dilation=9),
            _act(dim // 2),
            weight_norm(nn.Conv1d(dim // 2, dim, kernel_size=2 * stride, stride=stride, padding=stride // 2 + stride % 2)))

    def forward(self, x):
        _native_only("EncoderBlock")


def _init_weights(m):
    """facodec.py:21-24, as FACodecEncoder.reset_parameters applies it."""
    if isinstance(m, nn.Conv1d):
        nn.init.trunc_normal_(m.weight, std=0.02)
        nn.init.constant_(m.bias, 0)


class FACodecEncoder(_FACodecGenerator):
    """Drop-in for FACodecEncoder (facodec.py:157-194): the same constructor and parameter tree (``block.*``), so the
    released ``ns3_facodec_encoder.bin`` loads strictly.  ``forward(x)`` / ``inference(x)``: wav ``[B, 1, N]`` (any
    strides) -> ``[B, out_channels, F]`` fp32, F = ``frames(N)``."""

    kind = "facodec_encoder"

    def __init__(self, ngf=32, up_ratios=(2, 4, 5, 5), out_channels=1024):
        super().__init__()
        self.hop_length = int(np.prod(up_ratios))
        self.up_ratios = [int(u) for u in up_ratios]
        self.ngf, self.out_channels = int(ngf), int(out_channels)
        d_model = ngf
        block = [weight_norm(nn.Conv1d(1, d_model, kernel_size=7, padding=3))]
        for stride in up_ratios:
            d_model *= 2
            block.append(EncoderBlock(d_model, stride=stride))
        block += [_act(d_model), weight_norm(nn.Conv1d(d_model, out_channels, kernel_size=3, padding=1))]
        self.block = nn.Sequential(*block)
        self.enc_dim = d_model
        self.apply(_init_weights)

    # ---- NativeGenerator hooks -------------------------------------------------------
    def _input_channels(self):
        return 1

    def _c_config(self):
        if len(self.up_ratios) > _capi.AB_MAX_STAGES:
            raise ValueError("amphion_b200: too many up_ratios for the native encoder")
        c = _block_config(_capi.GEN_FACODEC_ENCODER, 1, self.ngf, self.up_ratios)
        c.trunk_out_channels = self.out_channels
        return c

    def frames(self, n_samples):
        """Output frames for n_samples input samples (0: a strided conv would have no output)."""
        t = int(n_samples)
        for s in self.up_ratios:
            pad = s // 2 + s % 2
            if t <= 0 or t + 2 * pad < 2 * s:
                return 0
            t = (t + 2 * pad - 2 * s) // s + 1
        return t

    # ---- served methods --------------------------------------------------------------
    def forward(self, x, out=None):
        """wav [B, 1, N] (any strides) -> [B, out_channels, F] fp32 on the wav's device.  ``out`` (beyond the reference
        signature): a contiguous fp32 [B, out_channels, F] tensor to write into."""
        if x.dim() != 3 or x.shape[1] != 1:
            raise ValueError(f"FACodecEncoder expects a waveform of shape [B, 1, N], got {tuple(x.shape)}")
        B, _, N = x.shape
        if B == 0 or N == 0:
            raise ValueError("amphion_b200: empty waveform batch")
        F = self.frames(N)
        if F <= 0:
            raise ValueError(f"FACodecEncoder: {N} samples are too short for up_ratios {self.up_ratios} (a strided "
                             f"conv's padded input would be shorter than its kernel)")
        _capi.require_cuda(x, "FACodecEncoder.forward")
        if x.dtype != torch.float32:
            x = x.float()
        with self._launch(x.device) as h:
            need = _capi.lib.ab_generator_workspace_bytes(h, B, N)
            ws = self._scratch(need, x.device)
            y = self._output(out, (B, self.out_channels, F), x.device)
            _capi.check(_capi.lib.ab_facodec_encode(h, _capi.ptr(x), B, N, _capi.shape_array(x.stride()), _capi.ptr(y),
                                                    ws, need, _capi.stream_ptr()), "ab_facodec_encode")
        return y

    def inference(self, x):
        return self.forward(x)


class FACodecRedecoder(_FACodecGenerator):
    """Drop-in for FACodecRedecoder (facodec.py:602-769): the same constructor and parameter tree
    (``{prosody,content,residual}_embs``, ``model.*``, ``timbre_linear``, ``timbre_cond_prosody_enc``), so the released
    ``ns3_facodec_redecoder.bin`` loads strictly.  Served natively (``AB_GEN_FACODEC_REDECODER``), in eval:

    - ``vq2emb(vq, speaker_embedding, use_residual=True)``: codes ``[n_q, B, T]`` (rows by position: prosody, content,
      residual; extra rows ignored) and the target speaker's embedding ``[B, 256]`` -> ``[B, 256, T]``;
    - ``inference(x, speaker_embedding)``: the decoder's FiLM and generator -> ``[B, 1, T * prod(up_ratios)]``.

    The transformer's style Linears read the speaker embedding itself; the reference reads the time mean of the
    embedding expanded over T, which equals it up to fp32 rounding of the sum."""

    kind = "facodec_redecoder"

    def __init__(self, in_channels=256, upsample_initial_channel=1280, up_ratios=(5, 5, 4, 2), vq_num_q_c=2,
                 vq_num_q_p=1, vq_num_q_r=3, vq_dim=256, codebook_size_prosody=10, codebook_size_content=10,
                 codebook_size_residual=10):
        super().__init__()
        if in_channels != 256 or vq_dim != 256:
            # the prosody transformer is 256 wide and its output is summed with the vq_dim-wide embeddings
            raise ValueError(f"amphion_b200: FACodecRedecoder needs in_channels == vq_dim == 256, the prosody "
                             f"transformer's width (got {in_channels}, {vq_dim})")
        self.hop_length = int(np.prod(up_ratios))
        self.up_ratios = [int(u) for u in up_ratios]
        self.in_channels, self.upsample_initial_channel = int(in_channels), int(upsample_initial_channel)
        self.vq_num_q_p, self.vq_num_q_c, self.vq_num_q_r = int(vq_num_q_p), int(vq_num_q_c), int(vq_num_q_r)
        self.vq_dim = int(vq_dim)
        self.codebook_size_prosody = codebook_size_prosody
        self.codebook_size_content = codebook_size_content
        self.codebook_size_residual = codebook_size_residual

        def embs(n, bits):
            out = nn.ModuleList()
            for _ in range(n):
                e = nn.Embedding(num_embeddings=2 ** bits, embedding_dim=vq_dim)
                e.weight.data.normal_(mean=0.0, std=1e-5)
                out.append(e)
            return out

        self.prosody_embs = embs(self.vq_num_q_p, codebook_size_prosody)
        self.content_embs = embs(self.vq_num_q_c, codebook_size_content)
        self.residual_embs = embs(self.vq_num_q_r, codebook_size_residual)
        _build_generator(self, in_channels, upsample_initial_channel, up_ratios)
        self.timbre_cond_prosody_enc = TransformerEncoder(use_cln=True)

    # ---- NativeGenerator hooks -------------------------------------------------------
    def _c_config(self):
        return _generator_config(self, _capi.GEN_FACODEC_REDECODER)

    # ---- served methods --------------------------------------------------------------
    def vq2emb(self, vq, speaker_embedding, use_residual=True):
        """codes [n_q, B, T] (integer, any strides), speaker_embedding [B, 256] -> [B, 256, T] fp32 on the codes'
        device (facodec.py:734-759)."""
        p, c, r = self.vq_num_q_p, self.vq_num_q_c, self.vq_num_q_r
        if not isinstance(vq, torch.Tensor) or vq.dim() != 3 or vq.is_floating_point() or vq.is_complex() \
                or vq.dtype == torch.bool:
            got = f"{vq.dtype} {tuple(vq.shape)}" if isinstance(vq, torch.Tensor) else type(vq).__name__
            raise ValueError(f"FACodecRedecoder.vq2emb expects integer codes [n_q, B, T], got {got}")
        n_q, B, T = vq.shape
        need = p + c + (r if use_residual else 0)
        if n_q < need:
            raise ValueError(f"FACodecRedecoder.vq2emb: {n_q} code rows, too few for {p} prosody, {c} content"
                             + (f" and {r} residual" if use_residual else "") + " rows")
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty code batch")
        spk = speaker_embedding
        if not isinstance(spk, torch.Tensor) or spk.dim() != 2 or tuple(spk.shape) != (B, self.in_channels):
            got = tuple(spk.shape) if isinstance(spk, torch.Tensor) else type(spk).__name__
            raise ValueError(f"FACodecRedecoder.vq2emb expects a speaker embedding of shape [{B}, {self.in_channels}], "
                             f"got {got}")
        if spk.device != vq.device:
            raise ValueError("FACodecRedecoder.vq2emb: the codes and the speaker embedding are on different devices")
        _capi.require_cuda(vq, "FACodecRedecoder.vq2emb")
        _refuse_training(self.timbre_cond_prosody_enc, "the prosody transformer", "dropout", _SERVED)
        n_pe = self.timbre_cond_prosody_enc.position_emb.pe.shape[0]
        if B > n_pe:
            raise ValueError(f"amphion_b200: batch {B} > {n_pe}, the rows of the prosody transformer's positional "
                             f"encoding (the reference fails there too)")
        vq = vq.long()
        _check_codes(self, vq, use_residual, "FACodecRedecoder", "embedding table")
        spk = spk.float()
        if spk.stride(1) != 1:
            spk = spk.contiguous()
        with self._launch(vq.device) as h:
            ws_bytes = _capi.lib.ab_facodec_redecoder_vq2emb_workspace_bytes(h, B, T)
            ws = self._scratch(ws_bytes, vq.device)
            out = torch.empty(B, self.in_channels, T, dtype=torch.float32, device=vq.device)
            _capi.check(_capi.lib.ab_facodec_redecoder_vq2emb(h, _capi.ptr(vq), _capi.shape_array(vq.stride()), n_q, B,
                                                              T, _capi.ptr(spk), spk.stride(0), int(bool(use_residual)),
                                                              _capi.ptr(out), ws, ws_bytes, _capi.stream_ptr()),
                        "ab_facodec_redecoder_vq2emb")
        return out

    def inference(self, x, speaker_embedding, out=None, tail_events=None):
        """x [B, 256, T] (any strides), speaker_embedding [B, 256] -> wav [B, 1, T * hop] fp32 (facodec.py:761-769).

        ``out`` / ``tail_events`` (beyond the reference signature) behave as in the other generators' forward."""
        return _inference(self, x, speaker_embedding, out, tail_events)

    def forward(self, *args, **kwargs):
        raise NotImplementedError(
            "amphion_b200: FACodecRedecoder.forward is not served: the reference builds the embedding sum as [B, T, d] "
            "and transposes it before timbre_norm, so it raises unless T == 256, and at T == 256 it normalises over "
            f"time and feeds [B, T, d] to conv_pre as channels.  Call vq2emb() and then inference(); {_SERVED}")


# ---- FACodec V2 (facodec.py:772-1199) ---------------------------------------------------------------------------------
_PROSODY_BINS = 20


class MelSpectrogram(_Holder):
    """Buffer holder for ns3_codec/melspec.py:39-102 as FACodecEncoderV2 builds it: ``mel_basis`` [num_mels, n_fft/2+1]
    (Slaney mel filterbank) and ``hann_window`` [win_size].  The transform runs on the native mel pipeline."""

    def __init__(self, n_fft, num_mels, sampling_rate, hop_size, win_size, fmin, fmax, center=False):
        super().__init__()
        from ..mel import librosa_mel_fn
        self.n_fft, self.hop_size, self.win_size = int(n_fft), int(hop_size), int(win_size)
        self.sampling_rate, self.num_mels, self.fmin, self.fmax, self.center = sampling_rate, num_mels, fmin, fmax, center
        self.register_buffer("mel_basis", librosa_mel_fn(sampling_rate, n_fft, num_mels, fmin, fmax).float())
        self.register_buffer("hann_window", torch.hann_window(win_size))


class FACodecEncoderV2(FACodecEncoder):
    """Drop-in for FACodecEncoderV2 (facodec.py:772-845): FACodecEncoder's parameter tree plus the buffers
    ``mel_transform.{mel_basis, hann_window}``, so ``ns3_facodec_encoder_v2.bin`` loads strictly.  ``forward`` /
    ``inference`` are FACodecEncoder's; ``get_prosody_feature(x)`` is served natively."""

    def __init__(self, ngf=32, up_ratios=(2, 4, 5, 5), out_channels=1024):
        super().__init__(ngf=ngf, up_ratios=up_ratios, out_channels=out_channels)
        self.mel_transform = MelSpectrogram(n_fft=1024, num_mels=80, sampling_rate=16000, hop_size=200, win_size=800,
                                            fmin=0, fmax=8000)

    def prosody_frames(self, n_samples):
        """Frames of get_prosody_feature for n_samples samples: (N + 2 pad - n_fft) // hop + 1, pad = (n_fft - hop) / 2."""
        mt = self.mel_transform
        pad = (mt.n_fft - mt.hop_size) // 2
        return (int(n_samples) + 2 * pad - mt.n_fft) // mt.hop_size + 1

    def get_prosody_feature(self, x):
        """wav [B, 1, N] (any strides) -> [B, 20, F] fp32 log-mel, the first 20 of the 80 mel rows (facodec.py:820-821):
        reflect pad (n_fft - hop) / 2, |STFT| with sqrt(re^2 + im^2 + 1e-9), the module's mel_basis rows, log(clamp(.,
        1e-5)).  Runs on the native STFT + mel pipeline with the module's own buffers."""
        from ..mel import native_stft_mel
        if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[1] != 1:
            got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
            raise ValueError(f"FACodecEncoderV2.get_prosody_feature expects a waveform of shape [B, 1, N], got {got}")
        mt = self.mel_transform
        pad = (mt.n_fft - mt.hop_size) // 2
        B, _, N = x.shape
        if B == 0:
            raise ValueError("amphion_b200: empty waveform batch")
        if N <= pad:
            raise ValueError(f"FACodecEncoderV2.get_prosody_feature: {N} samples are too few for the reflect pad of {pad} "
                             f"(the reference raises there too); it needs at least {pad + 1}")
        _capi.require_cuda(x, "FACodecEncoderV2.get_prosody_feature")
        basis = mt.mel_basis[:_PROSODY_BINS].to(device=x.device, dtype=torch.float32).contiguous()
        window = mt.hann_window.to(device=x.device, dtype=torch.float32).contiguous()
        with torch.no_grad():
            _, mel, _ = native_stft_mel(x[:, 0, :].float(), mt.n_fft, mt.hop_size, mt.win_size, window, basis, pad, 1e-9,
                                        clamp=1e-5)
        return mel


class FACodecDecoderV2(FACodecDecoder):
    """Drop-in for FACodecDecoderV2 (facodec.py:848-1199): FACodecDecoder's constructor and parameter tree plus
    ``melspec_linear`` (Linear 20 -> 256) and ``melspec_encoder`` (a 4-layer, 256-wide transformer), so
    ``ns3_facodec_decoder_v2.bin`` loads strictly.  Served natively, in eval:

    - ``forward(x, prosody_feature, vq=True)``: latent ``[B, 256, T]`` and prosody feature ``[B, 20, T]`` -> V1's
      5-tuple; the prosody group quantizes the prosody transformer's output (fp32 at every precision), the content
      group x, the residual group x - (prosody + content);
    - ``vq2emb(vq, use_residual=True)`` and ``inference(x, speaker_embedding)``: FACodecDecoder's."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.melspec_linear = nn.Linear(_PROSODY_BINS, 256)
        self.melspec_encoder = TransformerEncoder()
        self.apply(_init_weights)   # reset_parameters (facodec.py:1025): every Conv1d bias 0, as a fresh V2 decoder has

    def _c_config(self):
        c = super()._c_config()
        c.facodec_prosody_encoder = int(self._quantize_handle)
        return c

    def vq2emb(self, vq, use_residual=True):
        """codes [n_q, B, T] -> [B, in_channels, T] fp32 (facodec.py:1179-1190; FACodecDecoder.vq2emb's code path)."""
        return super().vq2emb(vq, use_residual_code=use_residual)

    def forward(self, x=None, prosody_feature=None, vq=True, get_vq=False, eval_vq=True, speaker_embedding=None,
                n_quantizers=None, quantized=None):
        """``vq=True``: x [B, 256, T] fp32 and prosody_feature [B, 20, T] (any strides) -> ``(outs [B, 256, T], qs int64
        [n_used, B, T], commit_loss zeros [n_used], quantized_buf [2 or 3 x [B, 256, T]], spk_embs [B, 256])`` on x's
        device, without autograd history (facodec.py:1064-1094 in eval).  ``n_quantizers = k`` keeps the first k layers
        of each group."""
        if get_vq:
            raise NotImplementedError(f"amphion_b200: FACodecDecoderV2.forward(get_vq=True) is not served; {_SERVED_V2}")
        if vq is not True:
            raise NotImplementedError(f"amphion_b200: the training branch of FACodecDecoderV2.forward (the predictors, "
                                      f"random residual masking) is not served; {_SERVED_V2}")
        if self.in_channels != 256:
            raise ValueError(f"amphion_b200: FACodecDecoderV2.forward(vq=True) needs in_channels == 256, the timbre "
                             f"encoder's width (got {self.in_channels})")
        if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[1] != self.in_channels:
            got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
            raise ValueError(f"FACodecDecoderV2.forward expects x of shape [B, {self.in_channels}, T], got {got}")
        pf = prosody_feature
        B, _, T = x.shape
        if not isinstance(pf, torch.Tensor) or pf.dim() != 3 or pf.shape[0] != B or pf.shape[1] != _PROSODY_BINS:
            got = tuple(pf.shape) if isinstance(pf, torch.Tensor) else type(pf).__name__
            raise ValueError(f"FACodecDecoderV2.forward expects a prosody feature of shape [{B}, {_PROSODY_BINS}, T], "
                             f"got {got}")
        if pf.shape[2] != T:
            # at hop 200 about a quarter of waveform lengths give one more encoder frame than mel frames
            raise ValueError(f"FACodecDecoderV2.forward: x has {T} frames and the prosody feature {pf.shape[2]}; they "
                             f"must match (the reference fails there too).  Trim the longer one to the shorter")
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty latent batch")
        if not x.is_cuda:
            raise NotImplementedError(f"amphion_b200: FACodecDecoderV2.forward(vq=True) needs a CUDA tensor (got "
                                      f"'{x.device}'); there is no CPU fallback; {_SERVED_V2}")
        if pf.device != x.device:
            raise ValueError("FACodecDecoderV2.forward: x and the prosody feature are on different devices")
        return self._quantize(x, pf, n_quantizers, eval_vq)
