"""Float64 restatement of the layer-normalised LSTM (ding/torch_utils/network/rnn.py:131-239, lstm_type='normal',
norm_type='LN') from its documented behaviour, for the tests.  Per layer l and step t:

    a   = LN(x_t Wx[l]; gamma_x, beta_x) + LN(h_{t-1} Wh[l]; gamma_h, beta_h) + bias[l]     (4H, biased variance, eps 1e-5)
    i, f, o, u = a[0:H], a[H:2H], a[2H:3H], a[3H:4H]
    c_t = sigmoid(f) c_{t-1} + sigmoid(i) tanh(u),   h_t = sigmoid(o) tanh(c_t)

Layer l's outputs h_1..h_T are layer l+1's inputs (after ``masks[l]``, a dropout mask already scaled by 1/(1-p), when
given).  Gradients come from torch's autograd over these float64 operations.
"""
import torch

EPS = 1e-5


def layer_norm(v, gamma, beta):
    mean = v.mean(-1, keepdim=True)
    var = ((v - mean)**2).mean(-1, keepdim=True)
    return (v - mean) / torch.sqrt(var + EPS) * gamma + beta


def forward(x, h0, c0, p, num_layers, masks=None):
    """x (T, B, I), h0 / c0 (L, B, H), p the parameters by their state_dict names -> (y (T, B, H), h_T, c_T (L, B, H))"""
    H = h0.shape[-1]
    hs, cs = [], []
    for l in range(num_layers):
        h, c = h0[l], c0[l]
        ys = []
        for t in range(x.shape[0]):
            a = (layer_norm(x[t] @ p['wx.%d' % l], p['norm.%d.weight' % (2 * l)], p['norm.%d.bias' % (2 * l)]) +
                 layer_norm(h @ p['wh.%d' % l], p['norm.%d.weight' % (2 * l + 1)], p['norm.%d.bias' % (2 * l + 1)]) +
                 p['bias'][l])
            i, f, o, u = a[:, :H], a[:, H:2 * H], a[:, 2 * H:3 * H], a[:, 3 * H:]
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(u)
            h = torch.sigmoid(o) * torch.tanh(c)
            ys.append(h)
        hs.append(h)
        cs.append(c)
        x = torch.stack(ys)
        if masks is not None and l < num_layers - 1:
            x = x * masks[l]
    return x, torch.stack(hs), torch.stack(cs)
