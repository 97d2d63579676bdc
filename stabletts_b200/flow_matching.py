"""Drop-in for the reference's ``models.flow_matching.CFMDecoder`` (models/flow_matching.py:11-100).

Same constructor, same ``forward(mu, mask, n_timesteps, temperature=1.0, c=None, solver=None,
cfg_kwargs=None)`` and ``cfg_wrapper``; ``.estimator`` is the drop-in ``Decoder``.  The whole ODE
solve (every estimator evaluation, CFG as a doubled batch, the Runge–Kutta updates) is ONE call
into the CUDA library, device-resident with no host synchronisation between steps.

Solver strings (webui.py:110): the fixed-grid ones (``'euler'``, ``'midpoint'``, ``'rk4'``) follow torchdiffeq's
published tableaux and run device-resident without any host synchronisation.  The reference's default
``solver=None`` (= ``'dopri5'``) is torchdiffeq's ADAPTIVE Dormand–Prince with ``rtol = atol = 1e-5``
(models/flow_matching.py:54): here it runs ``st_solve_adaptive`` — same published algorithm (FSAL
tableau, RMS mixed error norm, I-controller, dense output at t = 1), one 8-byte host read per step for
accept/reject exactly like torchdiffeq on a GPU.  torchdiffeq itself is absent and unpinned, so that
solver's parity is pinned only against ``oracle/adaptive_ref.py``; ``'bosh3'``, ``'fehlberg2'`` and
``'adaptive_heun'`` are further embedded tableaux on the same controller.  ``'dopri5_fixed'`` steps the
Dormand-Prince tableau on the caller's grid without error control (BASELINE.json cfg2's "dopri5-equiv").
``'implicit_adams'`` / ``'explicit_adams'`` raise ``ValueError`` (multistep methods are not built).
"""
from __future__ import annotations

import ctypes as C
import warnings

import torch
import torch.nn as nn

from . import _lib
from .estimator import Decoder

_METHODS = {"euler": _lib.ST_EULER, "midpoint": _lib.ST_MIDPOINT, "rk4": _lib.ST_RK4,
            "dopri5_fixed": _lib.ST_DOPRI5_FIXED}
# adaptive embedded Runge-Kutta tableaux of st_solve_adaptive_ex (webui.py:110 lists these strings)
_ADAPTIVE = {None: _lib.ST_ADAPT_DOPRI5, "dopri5": _lib.ST_ADAPT_DOPRI5, "bosh3": _lib.ST_ADAPT_BOSH3,
             "fehlberg2": _lib.ST_ADAPT_FEHLBERG2, "adaptive_heun": _lib.ST_ADAPT_HEUN}
_STAGES = {_lib.ST_ADAPT_DOPRI5: 6, _lib.ST_ADAPT_BOSH3: 3, _lib.ST_ADAPT_FEHLBERG2: 2, _lib.ST_ADAPT_HEUN: 1}
ST_ADAPTIVE = -1            # _method_id's answer for every adaptive solver; _ADAPTIVE picks the tableau


def _method_id(solver):
    if solver in _ADAPTIVE:
        return ST_ADAPTIVE
    if solver in _METHODS:
        return _METHODS[solver]
    if solver in ("implicit_adams", "explicit_adams"):
        raise ValueError(f"solver {solver!r} (torchdiffeq's fixed-grid Adams-Bashforth(-Moulton) multistep method) is not built "
                         f"in stabletts_b200; use one of {sorted(_METHODS)} (fixed grid) or "
                         f"{sorted(k for k in _ADAPTIVE if k)} / None (adaptive)")
    raise ValueError(f"solver {solver!r} is not supported; use one of {sorted(_METHODS)} (fixed grid) or "
                     f"{sorted(k for k in _ADAPTIVE if k)} / None (adaptive)")


class CFMDecoder(nn.Module):
    def __init__(self, noise_channels, cond_channels, hidden_channels, out_channels, filter_channels, n_heads, n_layers,
                 kernel_size, p_dropout, gin_channels):
        super().__init__()
        self.noise_channels = noise_channels
        self.cond_channels = cond_channels
        self.hidden_channels = hidden_channels
        self.out_channels = out_channels
        self.filter_channels = filter_channels
        self.gin_channels = gin_channels
        self.sigma_min = 1e-4
        self.last_solver_stats = None     # filled by the adaptive solver: accepted / rejected steps, NFE
        # argument order of Decoder differs from CFMDecoder's own (models/flow_matching.py:22)
        self.estimator = Decoder(noise_channels, cond_channels, hidden_channels, out_channels, filter_channels, p_dropout,
                                 n_layers, n_heads, kernel_size, gin_channels)

    @torch.inference_mode()
    def forward(self, mu, mask, n_timesteps, temperature=1.0, c=None, solver=None, cfg_kwargs=None, *, z=None):
        """models/flow_matching.py:24-55.  ``z`` (trailing, optional) injects the initial noise for
        tests; by default it is drawn exactly as the reference does, ``randn_like(mu) * temperature``
        from the global generator, UNMASKED (:45)."""
        est = self.estimator
        if mu.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        B, M, T = mu.shape
        if c is None:
            raise ValueError("c (speaker embedding, (B, gin_channels)) is required")
        if z is None:
            z = torch.randn_like(mu) * temperature                                   # :45
        z = est._f32c("z", z, (B, M, T)).clone()
        mu_ = est._f32c("mu", mu, (B, est.cond_channels, T))
        mask_ = est._f32c("mask", mask, (B, 1, T))
        c_ = est._f32c("c", c, (B, est.gin_channels))
        if B == 0 or T == 0:                     # empty batch / zero frames: odeint on an empty state returns it
            return z.to(mu.dtype)
        t_span = torch.linspace(0, 1, n_timesteps + 1, dtype=torch.float32)         # :46 (host copy of the grid)
        t_host = (C.c_float * (n_timesteps + 1))(*t_span.tolist())
        method = _method_id(solver)
        fc = fs = None
        strength = 1.0
        if cfg_kwargs is not None:                                                   # :49-52, :58-61
            fs = est._f32c("fake_speaker", cfg_kwargs["fake_speaker"].to(mu.device), (1, est.gin_channels))
            fc = est._f32c("fake_content", cfg_kwargs["fake_content"].to(mu.device), (1, est.cond_channels, 1))
            strength = float(cfg_kwargs["cfg_strength"])
        lib, h, stream = est._prepare(mu_, B, T, 0 if fc is None else 1)
        if method == ST_ADAPTIVE:                                                    # rtol = atol = 1e-5, :54
            stats = (C.c_int64 * 3)()
            tableau = _ADAPTIVE[solver]
            rc = lib.st_solve_adaptive_ex(h, tableau, z.data_ptr(), mu_.data_ptr(), mask_.data_ptr(), c_.data_ptr(),
                                          None if fc is None else fc.data_ptr(), None if fs is None else fs.data_ptr(),
                                          strength, float(t_span[0]), float(t_span[-1]), 1e-5, 1e-5, 100000, B, T, stream, stats)
            _lib.check(lib, h, rc, "st_solve_adaptive_ex")
            # torchdiffeq is absent/unpinned: this solver follows its published algorithm; parity with the package itself
            # is UNPINNED (oracle/adaptive_ref.py) -- the stats say so for callers that log them
            self.last_solver_stats = dict(solver=solver or "dopri5", accepted=int(stats[0]), rejected=int(stats[1]),
                                          nfe=int(stats[2]), stages_per_step=_STAGES[tableau], parity="unpinned (torchdiffeq absent)")
            return z.to(mu.dtype)
        rc = lib.st_solve(h, z.data_ptr(), mu_.data_ptr(), mask_.data_ptr(), c_.data_ptr(),
                          None if fc is None else fc.data_ptr(), None if fs is None else fs.data_ptr(),
                          strength, t_host, n_timesteps, method, B, T, stream)
        _lib.check(lib, h, rc, "st_solve")
        return z.to(mu.dtype)                                                        # trajectory[-1], :55

    @torch.inference_mode()
    def solve_host(self, mu, mask, n_timesteps, temperature=1.0, c=None, solver="euler", cfg_kwargs=None, *, z=None, out=None):
        """``forward`` for HOST tensors (the serving form: requests arrive in host memory): one ``st_solve_host`` call
        copies ``(z, mu, mask, c)`` host->device on the current stream of the module's device, runs the device-resident
        solve, copies the mel back and synchronises that stream.  Page-locked inputs (``tensor.pin_memory()``) are copied
        from directly, pageable ones are staged through a pinned buffer inside the library.  Fixed-grid solvers only.
        ``out``: optional (pinned) CPU tensor to receive the mel; by default a new pinned tensor is returned."""
        est = self.estimator
        dev = next(est.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: move the module with .to('cuda') (no CPU fallback)")
        if any(t is not None and t.device.type != "cpu" for t in (mu, mask, c, z)):
            raise RuntimeError("solve_host takes host tensors; use forward() for device tensors")
        method = _method_id(solver)
        if method == ST_ADAPTIVE:
            raise ValueError("solve_host runs the fixed-grid solvers (euler, midpoint, rk4, dopri5_fixed)")
        B, M, T = mu.shape
        if c is None:
            raise ValueError("c (speaker embedding, (B, gin_channels)) is required")
        if z is None:
            z = torch.randn_like(mu) * temperature                                   # :45
        if out is None:
            out = torch.empty((B, M, T), dtype=torch.float32).pin_memory() if B * T > 0 else torch.empty((B, M, T))
        if tuple(out.shape) != (B, M, T) or out.dtype != torch.float32 or not out.is_contiguous() or out.device.type != "cpu":
            raise ValueError("out must be a contiguous fp32 CPU tensor of shape (B, n_mel, T)")
        if B == 0 or T == 0:
            out.copy_(z.to(torch.float32).reshape(B, M, T))
            return out
        f32 = lambda t, shape: t.detach().to(torch.float32).reshape(shape).contiguous()
        mu_, mask_, c_ = f32(mu, (B, M, T)), f32(mask, (B, T)), f32(c, (B, est.gin_channels))
        z_ = f32(z, (B, M, T))                              # (no copy when z already is contiguous fp32: read in place)
        t_span = torch.linspace(0, 1, n_timesteps + 1, dtype=torch.float32)         # :46
        t_host = (C.c_float * (n_timesteps + 1))(*t_span.tolist())
        fc = fs = None
        strength = 1.0
        if cfg_kwargs is not None:
            fs = f32(cfg_kwargs["fake_speaker"].cpu(), (est.gin_channels,))
            fc = f32(cfg_kwargs["fake_content"].cpu(), (est.cond_channels,))
            strength = float(cfg_kwargs["cfg_strength"])
        with torch.cuda.device(dev):
            lib, h, stream = est._prepare(torch.empty(0, device=dev), B, T, 0 if fc is None else 1)
            rc = lib.st_solve_host_io(h, z_.data_ptr(), out.data_ptr(), mu_.data_ptr(), mask_.data_ptr(), c_.data_ptr(),
                                   None if fc is None else fc.data_ptr(), None if fs is None else fs.data_ptr(),
                                   strength, t_host, n_timesteps, method, B, T, stream)
        _lib.check(lib, h, rc, "st_solve_host_io")
        return out

    @torch.inference_mode()
    def cfg_wrapper(self, t, x, mask, mu, c, cfg_kwargs):
        """models/flow_matching.py:58-67 (kept for API parity; ``forward`` fuses the two branches into
        one doubled batch inside the library instead of calling this)."""
        fake_speaker = cfg_kwargs["fake_speaker"].repeat(x.size(0), 1)
        fake_content = cfg_kwargs["fake_content"].repeat(x.size(0), 1, x.size(-1))
        cfg_strength = cfg_kwargs["cfg_strength"]
        cond_output = self.estimator(t, x, mask, mu, c)
        uncond_output = self.estimator(t, x, mask, fake_content, fake_speaker)
        return uncond_output + cfg_strength * (cond_output - uncond_output)

    @torch.no_grad()
    def compute_loss(self, x1, mask, mu, c):
        """models/flow_matching.py:69-100, FORWARD VALUE ONLY: ``(loss, y)`` as the reference returns them from
        an ``eval()`` model under ``no_grad`` (a validation loss).  ``t`` and ``z`` are drawn exactly as the
        reference draws them (global generator, ``rand`` then ``randn_like``, :92-96); the mix, the estimator at
        per-sample ``t`` and the masked-sum reduction run in the CUDA library (``st_cfm_loss``).  Training —
        dropout and the backward pass — is outside this library's scope (SURVEY.md §8 row f3): in ``train()``
        mode this raises instead of silently returning a loss that cannot be differentiated."""
        if self.training:
            raise NotImplementedError("compute_loss in train() mode needs dropout + backward kernels, which are out of scope "
                                      "for the inference-only CUDA path; call .eval() for the validation loss, or train with "
                                      "the reference CFMDecoder and load the checkpoint here")
        est = self.estimator
        if mu.device.type != "cuda":
            raise RuntimeError("stabletts_b200 runs on CUDA (H100) only: there is no CPU fallback")
        B, M, T = mu.shape
        t = torch.rand([B, 1, 1], device=mu.device, dtype=mu.dtype)                  # :92
        t = 1 - torch.cos(t * 0.5 * torch.pi)                                        # :93
        z = torch.randn_like(x1)                                                     # :96
        x1_ = est._f32c("x1", x1, (B, M, T))
        z_ = est._f32c("z", z, (B, M, T))
        t_ = t.reshape(B).float().contiguous()
        mu_ = est._f32c("mu", mu, (B, est.cond_channels, T))
        mask_ = est._f32c("mask", mask, (B, 1, T))
        c_ = est._f32c("c", c, (B, est.gin_channels))
        y = torch.empty_like(x1_)
        loss = torch.empty((), device=mu.device, dtype=torch.float32)
        lib, h, stream = est._prepare(mu_, B, T, 0)
        rc = lib.st_cfm_loss(h, x1_.data_ptr(), z_.data_ptr(), t_.data_ptr(), mask_.data_ptr(), mu_.data_ptr(), c_.data_ptr(),
                             float(self.sigma_min), y.data_ptr(), loss.data_ptr(), B, T, stream)
        _lib.check(lib, h, rc, "st_cfm_loss")
        return loss.to(mu.dtype), y.to(mu.dtype)
