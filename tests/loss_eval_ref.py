"""Float64-capable restatements for held-out scoring (P2PModel.p2p_losses).  TEST INFRASTRUCTURE ONLY.

forward_losses_eval   models/p2p_model.py:185-257 with every module in eval mode (BatchNorm from its running statistics,
                      nothing updated), written on the oracle's layer functions (oracle/p2p_oracle.py) with training=False;
                      returns each term per row and the four scalars / seq_len derived from those rows
seq_losses_ref        what p2pvg_seq_losses computes from the buffers of an eval-mode forward, in float64
"""
import torch

from oracle import p2p_oracle as O


def _backbone(width):
    if width == "mlp":
        return (lambda p, xx: O.mlp_encoder_fwd(p, xx)), (lambda p, v, sk: O.mlp_decoder_fwd(p, v, sk))
    if width == "vgg":
        return (lambda p, xx: O.vgg_encoder_fwd(p, xx, training=False)), (lambda p, v, sk: O.vgg_decoder_fwd(p, v, sk, training=False))
    return (lambda p, xx: O.encoder_fwd(p, xx, width, training=False)), (lambda p, v, sk: O.decoder_fwd(p, v, sk, width, training=False))


def forward_losses_eval(state, x, opt, width, eps, probs):
    """The values P2PModel.forward(x) returns when every module is in eval mode (computed before its update).  state: module ->
    {key: tensor} (buffers are read, never written); x [T, B, ...]; eps [S, 2, B, z]; probs: the NumPy skip draw.
    Returns dict(losses=(mse, kld, cpc, align) / seq_len as floats, per_seq=[4, B] tensor of the rows' shares (element means
    over row b; kld: row b's KL sum / opt["batch_size"]), steps=[(i, time_until_cp, delta_time)])."""
    enc_fwd, dec_fwd = _backbone(width)
    enc, dec = state["encoder"], state["decoder"]
    fp, post, prior = state["frame_predictor"], state["posterior"], state["prior"]
    T, B = x.shape[0], x.shape[1]
    cp_ix = T - 1
    bs = opt["batch_size"] if opt.get("batch_size") is not None else B
    with torch.no_grad():
        hid_fp, hid_post, hid_prior = O.init_hidden(fp, B, x), O.init_hidden(post, B, x), O.init_hidden(prior, B, x)
        x_cp = x[cp_ix]
        global_z = enc_fwd(enc, x_cp)[0]
        sched = O.skip_schedule(T, probs, opt["skip_prob"], opt["n_past"])
        per = torch.zeros(4, B, dtype=x.dtype, device=x.device)
        h = h_pred = skip = None
        row_mse = lambda a, b: ((a - b) ** 2).reshape(B, -1).mean(1)
        for s, (i, tuc, dt) in enumerate(sched):
            if i > 1:   # p2p_model.py:224-225: h[0] is row 0 of the previous step's latent, broadcast
                per[3] += row_mse(h[0].expand_as(h_pred), h_pred)
            t_tuc = x.new_zeros(B, 1).fill_(tuc)
            t_dt = x.new_zeros(B, 1).fill_(dt)
            h_full = enc_fwd(enc, x[i - 1])
            h_target = enc_fwd(enc, x[i])[0]
            if opt["last_frame_skip"] or i <= opt["n_past"]:
                h, skip = h_full
            else:
                h = h_full[0]
            zt, mu, logvar = O.gaussian_lstm_fwd(post, hid_post, torch.cat([h_target, global_z, t_tuc, t_dt], 1), eps[s, 0])
            zt_p, mu_p, logvar_p = O.gaussian_lstm_fwd(prior, hid_prior, torch.cat([h, global_z, t_tuc, t_dt], 1), eps[s, 1])
            h_pred = O.lstm_fwd(fp, hid_fp, torch.cat([h, zt, t_tuc, t_dt], 1))
            x_pred = dec_fwd(dec, h_pred, skip)
            if i == cp_ix:
                h_pred_p = O.lstm_fwd(fp, hid_fp, torch.cat([h, zt_p, t_tuc, t_dt], 1))
                per[2] = row_mse(dec_fwd(dec, h_pred_p, skip), x_cp)
            per[0] += row_mse(x_pred, x[i])
            # misc/criterion.py:10-15 (O.kl_criterion) summed per row instead of over the whole batch
            s1, s2 = (logvar * 0.5).exp(), (logvar_p * 0.5).exp()
            per[1] += (torch.log(s2 / s1) + (torch.exp(logvar) + (mu - mu_p) ** 2) / (2 * torch.exp(logvar_p)) - 0.5).sum(1) / bs
        # the batch means of the reference's MSELoss terms are the means of the row means (equal row sizes); KL is the row sum
        losses = (per[0].mean(), per[1].sum(), per[2].mean(), per[3].mean())
    return dict(losses=tuple(float(v) / T for v in losses), per_seq=per / T, steps=sched)


def seq_losses_ref(rec, sigmoid, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, has_cpc, batch_size, seq_len):
    """float64 restatement of p2pvg_seq_losses (include/p2pvg_b200.h).  Returns (per_seq [4, B], out [4]) float64."""
    d = lambda t, n: t.reshape(-1)[:n].double()
    G = S + 1
    r = d(rec, G * B * E).reshape(G, B, E)
    if sigmoid:
        r = torch.sigmoid(r)
    tg = tgt[:G].long()
    nf = int(tg.max()) + 1
    xt = d(x, nf * B * E).reshape(nf, B, E)[tg]
    e2 = ((r - xt) ** 2).sum(2)                                    # [G, B]
    m1, l1, m2, l2 = (d(t, S * B * z).reshape(S, B, z) for t in (mu, lv, mu_p, lv_p))
    kl = (0.5 * (l2 - l1) + (l1.exp() + (m1 - m2) ** 2) / (2 * l2.exp()) - 0.5).sum(2)   # [S, B]
    nh = int(in_idx[:max(S - 1, 1)].max()) + 1
    Hv = d(H, nh * B * g).reshape(nh, B, g)
    hp = d(h_pred, G * B * g).reshape(G, B, g)
    al = torch.zeros(B, dtype=torch.float64, device=r.device)
    for s in range(S - 1):
        al += ((Hv[int(in_idx[s])][0].unsqueeze(0) - hp[s]) ** 2).sum(1)
    per = torch.stack([e2[:S].sum(0) / (E * seq_len), kl.sum(0) / (batch_size * seq_len),
                       (e2[S] / (E * seq_len)) if has_cpc else torch.zeros_like(al), al / (g * seq_len)])
    out = torch.stack([per[0].mean(), per[1].sum(), per[2].mean(), per[3].mean()])
    return per, out
