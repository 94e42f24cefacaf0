"""Oracle: SequentialRNNLM (LSTM cells) as a beam-search scorer (LM shallow fusion).  TEST INFRASTRUCTURE.

Reference: espnet2/lm/seq_rnn_lm.py:22-166 (Embedding -> nn.LSTM(batch_first) -> Linear; batch_score feeds the newest token with the
per-hypothesis (h, c) state).  The LSTM is restated with the gate equations of torch.nn.LSTM's documentation (gate order i, f, g, o):
    gates = x W_ih^T + b_ih + h W_hh^T + b_hh,  c' = sigmoid(f) c + sigmoid(i) tanh(g),  h' = sigmoid(o) tanh(c')
``batch_score(ys)`` runs the whole prefix from the zero state (states[0] is None in the reference), so it plugs into oracle.search's ``lm=``.
Weights: the SequentialRNNLM state_dict without the ESPnetLanguageModel ``lm.`` prefix ("encoder.weight", "rnn.weight_ih_l0", ...).
"""
import torch


class OracleRNNLM:
    def __init__(self, w, nlayers):
        self.w = {k: v.detach().float().cpu() for k, v in w.items()}
        self.n = nlayers
        if "decoder.weight" not in self.w:      # tie_weights: the decoder shares the embedding's parameter
            self.w["decoder.weight"] = self.w["encoder.weight"]
        self.H = self.w["rnn.weight_hh_l0"].shape[1]

    def _cell(self, x, h, c, k):
        w = self.w
        g = x @ w[f"rnn.weight_ih_l{k}"].t() + w[f"rnn.bias_ih_l{k}"] + h @ w[f"rnn.weight_hh_l{k}"].t() + w[f"rnn.bias_hh_l{k}"]
        i, f, gg, o = g.chunk(4, dim=-1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        return torch.sigmoid(o) * torch.tanh(c), c

    @torch.no_grad()
    def run(self, ys, state=None):
        """ys (n, len) int64 -> (log-probabilities of the next token after the last position (n, V), state (h, c) each [L][n][H])."""
        n = ys.shape[0]
        if state is None:
            h = [torch.zeros(n, self.H) for _ in range(self.n)]
            c = [torch.zeros(n, self.H) for _ in range(self.n)]
        else:
            h, c = [t.clone() for t in state[0]], [t.clone() for t in state[1]]
        emb = self.w["encoder.weight"][ys]
        for t in range(ys.shape[1]):
            x = emb[:, t]
            for k in range(self.n):
                h[k], c[k] = self._cell(x, h[k], c[k], k)
                x = h[k]
        logits = x @ self.w["decoder.weight"].t() + self.w["decoder.bias"]
        return torch.log_softmax(logits, dim=-1), (torch.stack(h), torch.stack(c))

    def batch_score(self, ys):
        return self.run(ys)[0]
