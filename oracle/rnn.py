"""Oracle: the RNN ASR model family on the CPU in float64 (or float32).  TEST INFRASTRUCTURE.

Restates, from the equations rather than by calling the reference modules:
  * VGG2L (legacy/nets/pytorch_backend/rnn/encoders.py): four 3x3 / stride 1 / pad 1 convs with ReLU, a 2x2 ceil-mode max-pool after the
    second and the fourth, lengths ceil(len / 2) per pool, output columns in (channel, freq) order;
  * RNNP (per layer a 1-layer (B)LSTM over the utterance's own frames, optional frame stride with lengths (len + 1) // sub, projection,
    tanh except after the last) and RNN (stacked (B)LSTM, l_last, tanh);
  * AttLoc and one RNNDecoder step (asr/decoder/rnn_decoder.py score): attention on the previous first-layer h, LSTMCells on
    [embed(y); c], output on z_L (or [z_L; c] with context_residual), log-softmax.
One utterance per call.  LSTM gate order i, f, g, o (torch.nn.LSTM's documentation).  Weights: the reference state_dict names without the
``encoder.`` / ``decoder.`` prefix.
"""
import torch
import torch.nn.functional as F


def _lstm_dir(x, wih, whh, bih, bhh, reverse):
    T, H = x.shape[0], whh.shape[1]
    h = x.new_zeros(H)
    c = x.new_zeros(H)
    ys = x.new_zeros(T, H)
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        g = wih @ x[t] + bih + whh @ h + bhh
        i, f, gg, o = g.chunk(4)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        ys[t] = h
    return ys


def lstm_layer(x, w, prefix, k, bidirectional):
    """One (B)LSTM layer k of an nn.LSTM's parameters under ``prefix`` over x (T, D) -> (T, ndir * H)."""
    outs = []
    for sfx in ("", "_reverse")[:2 if bidirectional else 1]:
        outs.append(_lstm_dir(x, w[f"{prefix}weight_ih_l{k}{sfx}"], w[f"{prefix}weight_hh_l{k}{sfx}"], w[f"{prefix}bias_ih_l{k}{sfx}"],
                              w[f"{prefix}bias_hh_l{k}{sfx}"], sfx == "_reverse"))
    return torch.cat(outs, dim=-1)


def vgg2l(x, w, prefix="enc.0."):
    """x (T, F) -> (ceil(ceil(T/2)/2), 128 * ceil(ceil(F/2)/2))."""
    y = x.view(1, 1, *x.shape)
    for a, b in (("conv1_1", "conv1_2"), ("conv2_1", "conv2_2")):
        for nm in (a, b):
            y = F.relu(F.conv2d(y, w[f"{prefix}{nm}.weight"], w[f"{prefix}{nm}.bias"], padding=1))
        y = F.max_pool2d(y, 2, stride=2, ceil_mode=True)
    return y[0].transpose(0, 1).reshape(y.shape[2], -1)


def rnn_encoder(x, w, conf, cls):
    """VGGRNNEncoder (cls "vgg_rnn") / RNNEncoder ("rnn") of one utterance x (T, F) -> (out (T', P), trace: [vgg?, projections after tanh])."""
    trace = []
    L, bidir = conf["num_layers"], conf.get("bidirectional", True)
    if cls == "vgg_rnn":
        x = vgg2l(x, w)
        trace.append(x)
        rnn = "enc.1."
        sub = [1] * (L + 1)
    else:
        rnn = "enc.0."
        s = conf.get("subsample", (2, 2, 1, 1))
        sub = [1] + (list(s)[:L] if s is not None else [])
        sub += [1] * (L + 1 - len(sub))
    if not conf.get("use_projection", True):
        for k in range(L):
            x = lstm_layer(x, w, rnn + "nbrnn.", k, bidir)
        return torch.tanh(x @ w[rnn + "l_last.weight"].t() + w[rnn + "l_last.bias"]), trace
    for i in range(L):
        y = lstm_layer(x, w, f"{rnn}{'birnn' if bidir else 'rnn'}{i}.", 0, bidir)
        if sub[i + 1] > 1:
            y = y[::sub[i + 1]]
        x = y @ w[f"{rnn}bt{i}.weight"].t() + w[f"{rnn}bt{i}.bias"]
        if i + 1 < L:
            x = torch.tanh(x)
        trace.append(x)
    return x, trace


class OracleRNNDecoder:
    """RNNDecoder.score for one hypothesis over one utterance's encoder output."""

    def __init__(self, w, num_layers, context_residual=False, scaling=2.0):
        self.w, self.L, self.ctx_res, self.scaling = w, num_layers, context_residual, scaling

    def att(self, enc, z0, a_prev):
        w = self.w
        T = enc.shape[0]
        if a_prev is None:
            a_prev = enc.new_full((T,), 1.0 / T)
        cw = w["att_list.0.loc_conv.weight"]                  # (chans, 1, 1, 2 filts + 1)
        filts = (cw.shape[-1] - 1) // 2
        conv = F.conv2d(a_prev.view(1, 1, 1, T), cw, padding=(0, filts))[0, :, 0].t()   # (T, chans)
        e = torch.tanh(conv @ w["att_list.0.mlp_att.weight"].t() + enc @ w["att_list.0.mlp_enc.weight"].t() + w["att_list.0.mlp_enc.bias"]
                       + w["att_list.0.mlp_dec.weight"] @ z0)
        e = e @ w["att_list.0.gvec.weight"][0] + w["att_list.0.gvec.bias"][0]
        a = torch.softmax(self.scaling * e, dim=0)
        return a @ enc, a

    def score(self, y, state, enc):
        """y: newest token id, state None or (z [L][H], c [L][H], a_prev (T,)), enc (T, E) -> (logp (V,), new state)."""
        w = self.w
        H = w["decoder.0.weight_hh"].shape[1]
        if state is None:
            z, c, a_prev = [enc.new_zeros(H) for _ in range(self.L)], [enc.new_zeros(H) for _ in range(self.L)], None
        else:
            z, c, a_prev = list(state[0]), list(state[1]), state[2]
        ctx, a = self.att(enc, z[0], a_prev)
        x = torch.cat([w["embed.weight"][y], ctx])
        nz, nc = [], []
        for k in range(self.L):
            g = w[f"decoder.{k}.weight_ih"] @ x + w[f"decoder.{k}.bias_ih"] + w[f"decoder.{k}.weight_hh"] @ z[k] + w[f"decoder.{k}.bias_hh"]
            i, f, gg, o = g.chunk(4)
            ck = torch.sigmoid(f) * c[k] + torch.sigmoid(i) * torch.tanh(gg)
            hk = torch.sigmoid(o) * torch.tanh(ck)
            nz.append(hk)
            nc.append(ck)
            x = hk
        out_in = torch.cat([x, ctx]) if self.ctx_res else x
        logits = w["output.weight"] @ out_in + w["output.bias"]
        return torch.log_softmax(logits, dim=0), (nz, nc, a)


def to(w, dtype=torch.float64):
    return {k: v.to(dtype) if torch.is_floating_point(v) else v for k, v in w.items()}

