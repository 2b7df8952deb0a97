"""CPU restatement (plain torch on fp32 CPU tensors) of the text side of the reference's evaluator: the RNN_ENCODER
forward in eval mode over a state_dict, the GloVe word lookups and padding mask, and prepare_cat_emb.  Every function
cites the reference lines it restates (paths under image_generation/ of the original project).  Each sample's sequence
is run on its own, with no packing, so the batch need not be sorted.  The tests compare it with the reference's own
RNN_ENCODER (tests/golden/reference/rnn_encoder_*.npz) and the CUDA path with it.
"""
import torch


def lstm_step(x, h, c, w_ih, w_hh, b_ih, b_hh):
    """One nn.LSTM cell step (gate order i, f, g, o): x (ninput,), h / c (H,) -> (h, c)."""
    gates = w_ih @ x + b_ih + w_hh @ h + b_hh
    i, f, g, o = gates.chunk(4)
    c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
    return torch.sigmoid(o) * torch.tanh(c), c


def rnn_encoder_forward(sd, captions, cap_lens, max_len):
    """RNN_ENCODER.forward (ref: model.py:145-179) after .eval(): dropout is the identity (model.py:151), the
    bidirectional one-layer LSTM runs over each caption's first cap_lens[b] tokens from a zero state (init_hidden,
    model.py:129-138; pack_padded_sequence), the backward direction from its last token; pad_packed_sequence and
    post_process_words (model.py:140-143) leave every column t >= cap_lens[b] of words_emb at zero up to max_len.
    Returns words_emb (B, 2H, max_len) and sent_emb (B, 2H) = [forward h_n, backward h_n] (model.py:170-174)."""
    emb = sd["encoder.weight"][captions]                      # (B, T, ninput)
    hid = sd["rnn.weight_hh_l0"].shape[1]
    b = captions.shape[0]
    words = torch.zeros(b, 2 * hid, max_len)
    sent = torch.zeros(b, 2 * hid)
    for d, sfx in enumerate(("", "_reverse")):
        w = [sd[f"rnn.{n}_l0{sfx}"] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        for i in range(b):
            n = int(cap_lens[i])
            h, c = torch.zeros(hid), torch.zeros(hid)
            for t in (range(n - 1, -1, -1) if d else range(n)):
                h, c = lstm_step(emb[i, t], h, c, *w)
                words[i, d * hid:(d + 1) * hid, t] = h
            sent[i, d * hid:(d + 1) * hid] = h
    return words, sent


def text_inputs(captions, glove_captions, glove, max_len):
    """evaluator.py:340-351: mask = (captions == 0)[:, :num_words] and glove_words_embs = glove_emb(glove_captions)
    [:, :num_words] transposed to (B, E, num_words), num_words = max_len."""
    mask = (captions == 0)[:, :max_len]
    glove_words = glove[glove_captions[:, :max_len]].transpose(1, 2)
    return glove_words, mask


def prepare_cat_emb(glove, cat_labels, cat_label_lens, order):
    """evaluator.py:148-164 (= trainer.py:227-241): one row per label of the length-sorted labels (load.py:305-355), the
    mean of its GloVe vectors when it has 1 or 2 tokens and zeros otherwise, then indexed by the resort indices."""
    raw = glove[cat_labels]                                   # (N, W, E)
    out = torch.zeros(raw.shape[0], raw.shape[2])
    for k in range(raw.shape[0]):
        n = int(cat_label_lens[k])
        if n == 1:
            out[k] = raw[k, 0]
        elif n == 2:
            out[k] = (raw[k, 0] + raw[k, 1]) / 2.
    return out[order]
