"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of the GRU-only scan ops of the decoupled RSSM
in `include/b200rl.h` (`b200rl_gru_scan_fwd` / `_bwd` / `_check` / `_workspace_bytes`), on top of the
`oracle/ops_emul.py::EmulOps` specification of every other op.  Same two uses: `-m gpu` tests compare the CUDA kernels
against it, and `-m "not gpu"` tests inject this object into `DV3Engine` (test double) to walk the decoupled schedule on
a GPU-less host.  The product never constructs it.
"""
from __future__ import annotations

import torch

from oracle.ops_emul import ACT_NONE, EmulOps

Tensor = torch.Tensor


class DecoupledEmulOps(EmulOps):
    def gru_scan_supported(self, dims: dict, backward: bool) -> bool:
        """b200rl_gru_scan_check without its shared-memory term (every R <= 1024 fits)"""
        return 1 <= dims["B"] <= 16 and dims["T"] >= 1 and dims["R"] % 2 == 0 and 2 <= dims["R"] <= 1024

    def gru_scan_workspace(self, T: int, B: int, R: int) -> Tensor:
        return torch.zeros(1, dtype=torch.int32)

    def gru_scan_fwd(self, dims: dict, eps: float, t: dict, workspace: Tensor):
        """All T steps of the GRU recurrence: g_pre holds x's share of the gate pre-activation on entry, the whole of it
        on return; fills g_ln, h_in and the h columns of latent."""
        T, B, R, off = dims["T"], dims["B"], dims["R"], dims["lat_off"]
        Wh = t["W_g"][:, :R]
        for i in range(T):
            s = slice(i * B, (i + 1) * B)
            prev = t["latent"][(i - 1) * B:i * B, off:off + R] if i > 0 else None
            self.mask_mix(prev, t["h0"], t["first"][s], t["h_in"][s])
            t["g_pre"][s].add_(t["h_in"][s] @ Wh.t())
            self.ln_act_fwd(t["g_pre"][s], t["lng_g"], t["lng_b"], eps, ACT_NONE, t["g_ln"][s])
            self.gru_gate_fwd(t["g_ln"][s], t["h_in"][s], t["latent"][s, off:off + R])

    def gru_scan_bwd(self, dims: dict, eps: float, t: dict, q: dict, workspace: Tensor):
        """BPTT of gru_scan_fwd: d_latent's h columns -> d_g_ln (the gradient of the LayerNorm's output, every step) and
        d_h0 (written)."""
        T, B, R, off = dims["T"], dims["B"], dims["R"], dims["lat_off"]
        Wh = t["W_g"][:, :R]
        carry = torch.zeros(B, R)
        d_pre, d_hin = torch.zeros(B, 3 * R), torch.zeros(B, R)
        q["d_h0"].zero_()
        for i in reversed(range(T)):
            s = slice(i * B, (i + 1) * B)
            dh = q["d_latent"][s, off:off + R] + carry
            self.gru_gate_bwd(t["g_ln"][s], t["h_in"][s], dh, q["d_g_ln"][s], d_hin)
            self.ln_act_bwd(t["g_pre"][s], t["lng_g"], t["lng_b"], eps, ACT_NONE, q["d_g_ln"][s], d_pre, None, None)
            d_hin.add_(d_pre @ Wh)
            self.mask_bwd(d_hin, t["first"][s], carry, q["d_h0"])
