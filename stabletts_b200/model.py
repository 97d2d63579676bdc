"""Drop-in for the reference's ``models.model.StableTTS`` (models/model.py:30-112): text + reference mel -> mel on this
library's kernels.  Same constructor, the same 189 ``state_dict`` keys at 80 mel channels (a reference checkpoint loads
with ``strict=True``), and ``synthesise`` with the reference's signature and return value:

    c = ref_encoder(y, None)                     MelStyleEncoder      (st_style_encoder_forward)
    x, mu_x, x_mask = encoder(x, c, x_lengths)   TextEncoder          (st_text_encoder_forward)
    logw = dp(x, x_mask, c)                      DurationPredictor    (st_duration_predictor_forward)
    mu_y, y_mask, attn = expand(logw, ...)       expand_by_durations  (st_align_lengths / st_align_expand)
    mel = decoder(mu_y, y_mask, ...)             CFMDecoder           (st_solve / st_solve_adaptive_ex)

The only host reads are the reference's own: ``y_lengths.max()`` (model.py:86) and the TextEncoder's token-id check.

``compute_losses`` is the VALUE of the training ``forward`` (model.py:114-178) in eval mode — the validation loss and
the forced alignment of a corpus under a trained model:

    c = ref_encoder(z, z_mask) / fake_speaker    MelStyleEncoder with a mask, cfg dropout mask drawn first (:138-141)
    x, mu_x, x_mask = encoder(x, c, x_lengths)   TextEncoder
    logw = dp(x, x_mask, c)                      DurationPredictor
    neg_cent = scores(y, mu_x)                   st_mas_scores                       (:150-155)
    attn, d, cum = maximum_path(neg_cent)        st_maximum_path, lengths from x_lengths / y_lengths   (:157-158)
    mu_y = expand(mu_x, cum)                     st_align_expand                     (:166-168)
    prior_loss, dur_loss                         st_mas_losses                       (:162-163, :175-176)
    diff_loss = decoder.compute_loss(...)        st_cfm_loss, mu_y / fake_content per the cfg mask (:171-173)

Training itself (dropout and the backward pass) is not built: ``forward`` raises."""
from __future__ import annotations

import torch
import torch.nn as nn

from . import monotonic_align
from .align import expand_by_cum, expand_by_durations
from .flow_matching import CFMDecoder
from .frontend import DurationPredictor, MelStyleEncoder
from .text_encoder import TextEncoder


class StableTTS(nn.Module):
    def __init__(self, n_vocab, mel_channels, hidden_channels, filter_channels, n_heads, n_enc_layers, n_dec_layers, kernel_size,
                 p_dropout, gin_channels):
        super().__init__()
        self.n_vocab = n_vocab
        self.mel_channels = mel_channels
        self.encoder = TextEncoder(n_vocab, mel_channels, hidden_channels, filter_channels, n_heads, n_enc_layers, kernel_size,
                                   p_dropout, gin_channels)
        self.ref_encoder = MelStyleEncoder(mel_channels, style_vector_dim=gin_channels, style_kernel_size=5, dropout=0.25)
        self.dp = DurationPredictor(hidden_channels, filter_channels, kernel_size, 0.5, gin_channels)
        self.decoder = CFMDecoder(mel_channels, mel_channels, hidden_channels, mel_channels, filter_channels, n_heads, n_dec_layers,
                                  kernel_size, p_dropout, gin_channels)
        # unconditional inputs of classifier-free guidance (model.py:43-44)
        self.fake_speaker = nn.Parameter(torch.zeros(1, gin_channels))
        self.fake_content = nn.Parameter(torch.zeros(1, mel_channels, 1))
        self.cfg_dropout = 0.2

    @torch.inference_mode()
    def synthesise(self, x, x_lengths, n_timesteps, temperature=1.0, y=None, length_scale=1.0, solver=None, cfg=1.0, *, z=None):
        """models/model.py:49-112.  Returns ``{"encoder_outputs": mu_y, "decoder_outputs": mel, "attn": path}`` of shapes
        (B, mel_channels, T_y), (B, mel_channels, T_y) and (B, 1, T_x, T_y).  ``cfg == 1.0`` runs without guidance.
        ``z`` (trailing, optional) injects the CFM's initial noise for tests; by default the decoder draws
        ``randn_like(mu_y) * temperature`` as the reference does."""
        if self.training:
            raise NotImplementedError("StableTTS.synthesise in train() mode would apply dropout, which the inference-only CUDA "
                                      "path does not build; call .eval() first")
        if y is None:
            raise ValueError("y (the reference mel, (B, mel_channels, T)) is required")
        c = self.ref_encoder(y, None)                                              # :79
        x, mu_x, x_mask = self.encoder(x, c, x_lengths)                            # :80
        logw = self.dp(x, x_mask, c)                                               # :81
        mu_y, y_mask, _, attn = expand_by_durations(logw, x_mask, mu_x, length_scale, return_attn=True)   # :83-95
        cfg_kwargs = None
        if cfg != 1.0:                                                             # :98-103
            cfg_kwargs = {"fake_speaker": self.fake_speaker, "fake_content": self.fake_content, "cfg_strength": cfg}
        decoder_outputs = self.decoder(mu_y, y_mask, n_timesteps, temperature, c, solver, cfg_kwargs, z=z)
        return {"encoder_outputs": mu_y, "decoder_outputs": decoder_outputs, "attn": attn}

    def forward(self, x, x_lengths, y, y_lengths, z, z_lengths):
        raise NotImplementedError("StableTTS.forward trains (dropout, backward), which this CUDA path does not build: train "
                                  "with the reference StableTTS and load its checkpoint here (load_state_dict(strict=True)); "
                                  "compute_losses(...) gives the forward's losses and alignment in eval mode")

    @torch.no_grad()
    def compute_losses(self, x, x_lengths, y, y_lengths, z, z_lengths):
        """The value of models/model.py:114-178 in eval mode: ``(dur_loss, diff_loss, prior_loss, attn)`` with attn
        (B, T_x, T_y) as the reference returns it.  The global generator is consumed in the reference's order: the cfg
        dropout mask ``torch.rand(B, 1) > cfg_dropout`` (:138), then ``compute_loss``'s ``t`` and ``z`` (flow_matching.py:90-94).
        x (B, T_x) token ids, y (B, n_mel, T_y) target mel, z (B, n_mel, T_z) the reference-encoder slice, with their
        lengths.  In ``train()`` mode this raises: dropout and the backward pass are not built."""
        if self.training:
            raise NotImplementedError("StableTTS.compute_losses in train() mode would need dropout and the backward pass, which "
                                      "this CUDA path does not build; call .eval() for the validation loss")
        if not isinstance(y, torch.Tensor) or y.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        B, M, Ty = y.shape
        if M != self.mel_channels or tuple(z.shape[:2]) != (B, M) or tuple(x.shape[:1]) != (B,):
            raise ValueError(f"y (B, {self.mel_channels}, T_y), z (B, {self.mel_channels}, T_z) and x (B, T_x) must share B; got "
                             f"{tuple(y.shape)}, {tuple(z.shape)}, {tuple(x.shape)}")
        dev = y.device
        z_lengths = torch.as_tensor(z_lengths, device=dev)
        z_mask = (torch.arange(z.size(2), device=dev)[None] < z_lengths[:, None]).unsqueeze(1).to(z.dtype)     # :137
        cfg_mask = torch.rand(B, 1, device=dev) > self.cfg_dropout                                            # :138
        c = self.ref_encoder(z, z_mask) * cfg_mask + ~cfg_mask * self.fake_speaker.repeat(B, 1)                # :141
        x, mu_x, x_mask = self.encoder(x, c, x_lengths)                                                        # :143
        logw = self.dp(x, x_mask, c)                                                                           # :144
        Tx = mu_x.shape[2]
        xl = torch.as_tensor(x_lengths, device=dev).to(torch.int64).contiguous()
        yl = torch.as_tensor(y_lengths, device=dev).to(torch.int64).contiguous()
        y_ = y.detach().to(torch.float32).contiguous()
        neg_cent = monotonic_align.scores(y_, mu_x)                                                            # :150-155
        ws = monotonic_align.workspace(B, Ty, Tx, dev)
        path, dur, cum = monotonic_align.search(neg_cent, x_lengths=xl, y_lengths=yl, ws=ws)                   # :157-158
        x_mask_ = x_mask.reshape(B, Tx).contiguous()
        mu_y, y_mask, _ = expand_by_cum(mu_x, x_mask_, cum, yl, Ty)                                            # :136, :166-168
        prior_loss, dur_loss = monotonic_align.losses(y_, mu_y, y_mask, logw.reshape(B, Tx).contiguous(), x_mask_, dur, xl, ws)
        keep = cfg_mask.unsqueeze(-1)                                                                          # :171-172
        mu_y_masked = mu_y * keep + ~keep * self.fake_content.repeat(B, 1, Ty)
        diff_loss, _ = self.decoder.compute_loss(y, y_mask, mu_y_masked, c)                                    # :173
        return dur_loss, diff_loss, prior_loss, path.transpose(1, 2)                                           # :166, :178
