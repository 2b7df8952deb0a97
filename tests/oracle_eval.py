"""Eval-mode restatement of the generator forward for the tests: the oracle's G_NET forward
(oracle/objgan_oracle.py g_net_forward) with every BatchNorm in eval mode (ref: nn.BatchNorm{1,2}d after
netG.eval(), evaluator.py:110) -- normalised with the running statistics, which stay untouched.

The oracle's blocks reach BatchNorm through its module-level ``batch_norm_train``; ``g_net_forward_eval`` swaps in
``batch_norm_eval`` for the duration of one call, so the eval-mode network is the oracle's own composition."""
import contextlib

import torch.nn.functional as F

from oracle import objgan_oracle as O


def batch_norm_eval(x, sd, prefix):
    """nn.BatchNorm{1,2}d in eval mode: F.batch_norm(training=False) with the running statistics."""
    return F.batch_norm(x, sd[prefix + ".running_mean"], sd[prefix + ".running_var"], sd[prefix + ".weight"],
                        sd[prefix + ".bias"], False, O.BN_MOMENTUM, O.EPS_NORM)


@contextlib.contextmanager
def _eval_batch_norm():
    saved = O.batch_norm_train
    O.batch_norm_train = lambda x, sd, prefix, update=True: batch_norm_eval(x, sd, prefix)
    try:
        yield
    finally:
        O.batch_norm_train = saved


def g_net_forward_eval(sd, inp, **kw):
    """O.g_net_forward with eval-mode BatchNorm; ``sd`` is not modified."""
    with _eval_batch_norm():
        return O.g_net_forward(sd, inp, update=False, **kw)
