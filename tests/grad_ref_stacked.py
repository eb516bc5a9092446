"""Float64 reference of a stacked LSTM stem (torch.nn.LSTM with num_layers > 1), built from grad_ref.lstm."""
from grad_ref import lstm


def lstm_stack(x, h0, c0, layers):
    """torch.nn.LSTM(num_layers = len(layers), batch_first, dropout 0) as ``grad_ref.lstm()`` per layer: layer 0 reads
    ``x``, layer k > 0 reads layer k-1's ``h``.  ``layers``: per layer (w_ih, w_hh, b_ih, b_hh); h0 / c0: per-layer lists
    of [B, H] (or None: zeros).  -> the list of per-layer ``lstm()`` dicts (the top layer's ``h`` is the stem output)."""
    out = []
    for k, w in enumerate(layers):
        r = lstm(x, None if h0 is None else h0[k], None if c0 is None else c0[k], *w)
        out.append(r)
        x = r['h']
    return out
