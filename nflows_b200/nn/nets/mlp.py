"""Multi-layer perceptron conditioner (reference nflows/nn/nets/mlp.py:9-68)."""
import numpy as np
import torch
from torch import nn
from torch.nn import functional as F


class MLP(nn.Module):
    """Linear/activation stack on flattened inputs of shape `in_shape`, producing `out_shape`."""

    def __init__(self, in_shape, out_shape, hidden_sizes, activation=F.relu, activate_output=False):
        super().__init__()
        self._in_shape = torch.Size(in_shape)
        self._out_shape = torch.Size(out_shape)
        self._hidden_sizes = hidden_sizes
        self._activation = activation
        self._activate_output = activate_output
        if len(hidden_sizes) == 0:
            raise ValueError("List of hidden sizes can't be empty.")
        self._input_layer = nn.Linear(int(np.prod(in_shape)), hidden_sizes[0])
        self._hidden_layers = nn.ModuleList(
            [nn.Linear(a, b) for a, b in zip(hidden_sizes[:-1], hidden_sizes[1:])])
        self._output_layer = nn.Linear(hidden_sizes[-1], int(np.prod(out_shape)))

    def forward(self, inputs, context=None):
        if inputs.shape[1:] != self._in_shape:
            raise ValueError("Expected inputs of shape {}, got {}.".format(self._in_shape, inputs.shape[1:]))
        t = self._activation(self._input_layer(inputs.reshape(-1, int(np.prod(self._in_shape)))))
        for layer in self._hidden_layers:
            t = self._activation(layer(t))
        t = self._output_layer(t)
        if self._activate_output:
            t = self._activation(t)
        return t.reshape(-1, *self._out_shape)

    def dense_chain(self, context=None):
        """[(weight, bias, act_in, act_out, residual)] with the activation's code (dense.activation_code) in the act slots, or
        None when this net needs the generic torch path."""
        from ... import dense as D
        act = D.native_activation(self._activation)
        if context is not None or act is None or len(self._in_shape) != 1 or len(self._out_shape) != 1:
            return None
        layers = [self._input_layer] + list(self._hidden_layers)
        chain = [(l.weight, l.bias, 0, act, None) for l in layers]
        chain.append((self._output_layer.weight, self._output_layer.bias, 0, act if self._activate_output else 0, None))
        return chain
