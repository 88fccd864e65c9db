"""TEST INFRASTRUCTURE — executable specification (plain fp32 torch, CPU) of the recurrent-PPO C-ABI ops in
`include/b200rl.h` (`b200rl_ppo_loss_masked`, `b200rl_lstm_seq_fwd`, `b200rl_lstm_seq_bwd`), on top of the
`oracle/ops_emul.py::EmulOps` specification of every other op.  Same two uses: `-m gpu` tests compare each CUDA kernel
against the method of the same name, and `-m "not gpu"` tests inject this object into `RecurrentPPOEngine` (test
double) to walk the engine's schedule on a GPU-less host.  The product never constructs it.
"""
from __future__ import annotations

import torch

from oracle.ops_emul import EmulOps


class RecurrentEmulOps(EmulOps):
    def ppo_loss_masked(self, head, actions, old_logp, adv, values, old_values, returns, mask, dhead, dvalues, losses,
                        head_dims, is_continuous, clip_vloss, normalize_adv, clip_coef, vf_coef, ent_coef):
        """ppo_loss over the rows with mask != 0 (ppo_recurrent.py:77-101): advantages normalised only when more
        than one row is kept; the other rows get zero gradients; no kept row -> zero losses and gradients."""
        keep = (mask.reshape(-1) != 0).nonzero().reshape(-1)
        dhead.zero_(), dvalues.zero_()
        if keep.numel() == 0:
            losses.zero_()
            return
        n = keep.numel()
        gh, gv = torch.zeros(n, head.shape[1]), torch.zeros(n)
        self.ppo_loss(head[keep], actions[keep], old_logp[keep], adv[keep], values[keep], old_values[keep],
                      returns[keep], gh, gv, losses, head_dims, is_continuous, clip_vloss, normalize_adv and n > 1,
                      clip_coef, vf_coef, ent_coef)
        dhead[keep], dvalues[keep] = gh, gv

    # ---- recurrent PPO: single-layer LSTM over padded sequences (csrc/lstm.cu)
    def lstm_seq_fwd(self, xw, W_hh, h0, c0, lengths, out, gates=None, cs=None, hT=None, cT=None):
        """torch nn.LSTM step (gates i, f, g, o) for t < lengths[b]; padded steps: out 0, state kept."""
        T, B, G = xw.shape
        H = G // 4
        h, c = h0.reshape(B, H).clone(), c0.reshape(B, H).clone()
        o_, g_, c_ = out.view(T, B, H), None if gates is None else gates.view(T, B, G), None if cs is None else cs.view(T, B, H)
        for t in range(T):
            z = xw[t] + h @ W_hh.t()
            i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
            cn = f * c + i * g
            hn = o * torch.tanh(cn)
            valid = (t < lengths.reshape(-1).long()).unsqueeze(-1)
            c, h = torch.where(valid, cn, c), torch.where(valid, hn, h)
            o_[t] = torch.where(valid, hn, torch.zeros_like(hn))
            if g_ is not None:
                g_[t] = torch.where(valid, torch.cat((i, f, g, o), -1), torch.zeros_like(z))
                c_[t] = torch.where(valid, cn, torch.zeros_like(cn))
        if hT is not None:
            hT.view(B, H).copy_(h)
        if cT is not None:
            cT.view(B, H).copy_(c)

    def lstm_seq_bwd(self, d_out, W_hh, gates, cs, c0, lengths, d_gates):
        """d_gates = gradient w.r.t. the pre-activation gates (BPTT); zero at padded steps; no gradient to h0/c0."""
        T, B, G = d_gates.shape
        H = G // 4
        gt, ct, do = gates.view(T, B, G), cs.view(T, B, H), d_out.view(T, B, H)
        dg_out = d_gates.view(T, B, G)
        dh, dc = torch.zeros(B, H), torch.zeros(B, H)
        for t in reversed(range(T)):
            valid = (t < lengths.reshape(-1).long()).unsqueeze(-1)
            i, f, g, o = gt[t, :, :H], gt[t, :, H:2 * H], gt[t, :, 2 * H:3 * H], gt[t, :, 3 * H:]
            cp = ct[t - 1] if t > 0 else c0.reshape(B, H)
            tc = torch.tanh(ct[t])
            dht = do[t] + dh
            dct = dc + dht * o * (1 - tc * tc)
            dg = torch.cat((dct * g * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - g * g), dht * tc * o * (1 - o)), -1)
            dg = torch.where(valid, dg, torch.zeros_like(dg))
            dg_out[t] = dg
            dc = torch.where(valid, dct * f, torch.zeros_like(dct))
            dh = dg @ W_hh
