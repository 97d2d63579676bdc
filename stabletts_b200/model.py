"""Drop-in for the reference's ``models.model.StableTTS`` (models/model.py:30-112): text + reference mel -> mel on this
library's kernels.  Same constructor, the same 189 ``state_dict`` keys at 80 mel channels (a reference checkpoint loads
with ``strict=True``), and ``synthesise`` with the reference's signature and return value:

    c = ref_encoder(y, None)                     MelStyleEncoder      (st_style_encoder_forward)
    x, mu_x, x_mask = encoder(x, c, x_lengths)   TextEncoder          (st_text_encoder_forward)
    logw = dp(x, x_mask, c)                      DurationPredictor    (st_duration_predictor_forward)
    mu_y, y_mask, attn = expand(logw, ...)       expand_by_durations  (st_align_lengths / st_align_expand)
    mel = decoder(mu_y, y_mask, ...)             CFMDecoder           (st_solve / st_solve_adaptive_ex)

The only host reads are the reference's own: ``y_lengths.max()`` (model.py:86) and the TextEncoder's token-id check.
Training (``forward``: monotonic alignment search, dropout, backward) is not built."""
from __future__ import annotations

import torch
import torch.nn as nn

from .align import expand_by_durations
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
        raise NotImplementedError("StableTTS.forward computes the training losses (monotonic alignment search, dropout, "
                                  "backward), which the inference-only CUDA path does not build: train with the reference "
                                  "StableTTS and load its checkpoint here (load_state_dict(strict=True))")
