"""Residual conditioner networks (reference nflows/nn/nets/resnet.py:9-205).

`ResidualNet` is the conditioner of the coupling transforms on the hot path.  When it is the plain no
batch-norm / no active dropout configuration with an activation the kernels run (dense.activation_code),
`dense_chain()` describes it as a list of dense layers so the coupling can execute it with `nfk_linear` launches
(bias, activation and the residual add are fused into the GEMM epilogues)."""
import torch
from torch import nn
from torch.nn import functional as F
from torch.nn import init


class ResidualBlock(nn.Module):
    """Pre-activation residual block on feature vectors: x + W2 drop(act(bn(W1 act(bn(x)))))."""

    def __init__(self, features, context_features, activation=F.relu, dropout_probability=0.0, use_batch_norm=False,
                 zero_initialization=True):
        super().__init__()
        self.activation = activation
        self.use_batch_norm = use_batch_norm
        if use_batch_norm:
            self.batch_norm_layers = nn.ModuleList([nn.BatchNorm1d(features, eps=1e-3) for _ in range(2)])
        if context_features is not None:
            self.context_layer = nn.Linear(context_features, features)
        self.linear_layers = nn.ModuleList([nn.Linear(features, features) for _ in range(2)])
        self.dropout = nn.Dropout(p=dropout_probability)
        if zero_initialization:
            init.uniform_(self.linear_layers[-1].weight, -1e-3, 1e-3)
            init.uniform_(self.linear_layers[-1].bias, -1e-3, 1e-3)

    def forward(self, inputs, context=None):
        t = inputs
        if self.use_batch_norm:
            t = self.batch_norm_layers[0](t)
        t = self.linear_layers[0](self.activation(t))
        if self.use_batch_norm:
            t = self.batch_norm_layers[1](t)
        t = self.linear_layers[1](self.dropout(self.activation(t)))
        if context is not None:
            t = F.glu(torch.cat((t, self.context_layer(context)), dim=1), dim=1)
        return inputs + t


class ResidualNet(nn.Module):
    """Linear -> num_blocks residual blocks -> Linear, on feature vectors."""

    def __init__(self, in_features, out_features, hidden_features, context_features=None, num_blocks=2,
                 activation=F.relu, dropout_probability=0.0, use_batch_norm=False):
        super().__init__()
        self.hidden_features = hidden_features
        self.context_features = context_features
        first_in = in_features if context_features is None else in_features + context_features
        self.initial_layer = nn.Linear(first_in, hidden_features)
        self.blocks = nn.ModuleList([
            ResidualBlock(features=hidden_features, context_features=context_features, activation=activation,
                          dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)
            for _ in range(num_blocks)
        ])
        self.final_layer = nn.Linear(hidden_features, out_features)

    def forward(self, inputs, context=None):
        t = self.initial_layer(inputs if context is None else torch.cat((inputs, context), dim=1))
        for block in self.blocks:
            t = block(t, context=context)
        return self.final_layer(t)

    def _context_parts(self):
        """Slices of the parameters the context path multiplies separately, as persistent tensors (the split pairs are cached on
        them): W0[:, :d_id]; W0[:, d_id:] and every block's context_layer weight zero padded to a multiple of 8 columns (TMA
        rows) next to their unpadded copies.  Rebuilt when a parameter or the cache epoch changes."""
        from ... import dense as D

        def build():
            c = self.context_features
            pad = (c + 7) // 8 * 8

            def padded(w):
                w = w.detach()
                out = w.new_zeros(w.shape[0], pad)
                out[:, :c] = w
                return out, w.contiguous()

            w0 = self.initial_layer.weight.detach()
            d_id = w0.shape[1] - c
            return {"w0a": w0[:, :d_id].contiguous(), "w0b": padded(w0[:, d_id:]),
                    "gates": [padded(b.context_layer.weight) for b in self.blocks], "pad": pad}
        return D.derived(self, "_ctx_parts", [self.initial_layer.weight] + [b.context_layer.weight for b in self.blocks], build)

    def dense_chain(self, context=None):
        """[(weight, bias, act_in, act_out, residual)] or None when this net needs the generic torch path; the act slots hold the
        code of the blocks' activation (dense.activation_code), 0 for none.
        residual: None, or "skip" = add the block input.  With a context (2-D fp32, context_features columns) the list is a
        dense.Chain whose layers also carry the tokens "ctx_init" / "glu_skip" (resnet.py:36-100 of the reference)."""
        if (context is None) != (self.context_features is None):
            return None
        if context is not None and (context.dim() != 2 or context.shape[1] != self.context_features
                                    or context.dtype != torch.float32):
            return None
        from ... import dense as D
        acts = [D.native_activation(block.activation) for block in self.blocks]
        for block, act in zip(self.blocks, acts):
            if block.use_batch_norm or act is None:
                return None
            if block.dropout.p > 0.0 and block.training:
                return None
        if context is None:
            chain = [(self.initial_layer.weight, self.initial_layer.bias, 0, 0, None)]
            for block, act in zip(self.blocks, acts):
                l0, l1 = block.linear_layers
                chain.append((l0.weight, l0.bias, act, act, None))
                chain.append((l1.weight, l1.bias, 0, 0, "skip"))
            chain.append((self.final_layer.weight, self.final_layer.bias, 0, 0, None))
            return chain
        parts = self._context_parts()
        layers = [(parts["w0a"], None, 0, 0, "ctx_init")]
        gates = {}
        for block, act, (wg_pad, wg) in zip(self.blocks, acts, parts["gates"]):
            l0, l1 = block.linear_layers
            layers.append((l0.weight, l0.bias, act, act, None))
            gates[len(layers)] = (wg_pad, block.context_layer.bias, wg)
            layers.append((l1.weight, l1.bias, 0, 0, "glu_skip"))
        layers.append((self.final_layer.weight, self.final_layer.bias, 0, 0, None))
        return D.Chain(layers, context, (parts["w0b"][0], self.initial_layer.bias, parts["w0b"][1]), gates, parts["pad"])


class ConvResidualBlock(nn.Module):
    def __init__(self, channels, context_channels=None, activation=F.relu, dropout_probability=0.0, use_batch_norm=False,
                 zero_initialization=True):
        super().__init__()
        self.activation = activation
        if context_channels is not None:
            self.context_layer = nn.Conv2d(in_channels=context_channels, out_channels=channels, kernel_size=1, padding=0)
        self.use_batch_norm = use_batch_norm
        if use_batch_norm:
            self.batch_norm_layers = nn.ModuleList([nn.BatchNorm2d(channels, eps=1e-3) for _ in range(2)])
        self.conv_layers = nn.ModuleList([nn.Conv2d(channels, channels, kernel_size=3, padding=1) for _ in range(2)])
        self.dropout = nn.Dropout(p=dropout_probability)
        if zero_initialization:
            init.uniform_(self.conv_layers[-1].weight, -1e-3, 1e-3)
            init.uniform_(self.conv_layers[-1].bias, -1e-3, 1e-3)

    def forward(self, inputs, context=None):
        t = inputs
        if self.use_batch_norm:
            t = self.batch_norm_layers[0](t)
        t = self.conv_layers[0](self.activation(t))
        if self.use_batch_norm:
            t = self.batch_norm_layers[1](t)
        t = self.conv_layers[1](self.dropout(self.activation(t)))
        if context is not None:
            t = F.glu(torch.cat((t, self.context_layer(context)), dim=1), dim=1)
        return inputs + t


class ConvResidualNet(nn.Module):
    """1x1 conv -> residual 3x3 blocks -> 1x1 conv (image conditioner; torch/cuDNN path, off the hot path)."""

    def __init__(self, in_channels, out_channels, hidden_channels, context_channels=None, num_blocks=2,
                 activation=F.relu, dropout_probability=0.0, use_batch_norm=False):
        super().__init__()
        self.context_channels = context_channels
        self.hidden_channels = hidden_channels
        first_in = in_channels if context_channels is None else in_channels + context_channels
        self.initial_layer = nn.Conv2d(in_channels=first_in, out_channels=hidden_channels, kernel_size=1, padding=0)
        self.blocks = nn.ModuleList([
            ConvResidualBlock(channels=hidden_channels, context_channels=context_channels, activation=activation,
                              dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)
            for _ in range(num_blocks)
        ])
        self.final_layer = nn.Conv2d(hidden_channels, out_channels, kernel_size=1, padding=0)

    def forward(self, inputs, context=None):
        t = self.initial_layer(inputs if context is None else torch.cat((inputs, context), dim=1))
        for block in self.blocks:
            t = block(t, context)
        return self.final_layer(t)

    def _dense_parts(self):
        """The convolution weights as dense-layer matrices on pixel rows, persistent tensors rebuilt when a parameter (or the
        cache epoch) changes: 1x1 kernels [out, in] (the initial one zero padded to a multiple of 8 input columns), 3x3 kernels
        [out, 9*in] in (ky, kx, c) order -- the column order of kernels.im2col3x3."""
        from ... import dense as D
        convs = [self.initial_layer] + [c for b in self.blocks for c in b.conv_layers] + [self.final_layer]

        def build():
            w0 = self.initial_layer.weight.detach().flatten(1)
            pad = (w0.shape[1] + 7) // 8 * 8
            first = w0.new_zeros(w0.shape[0], pad)
            first[:, :w0.shape[1]] = w0
            mats = [first]
            for b in self.blocks:
                for c in b.conv_layers:
                    mats.append(c.weight.detach().permute(0, 2, 3, 1).reshape(c.weight.shape[0], -1).contiguous())
            mats.append(self.final_layer.weight.detach().flatten(1).contiguous())
            return mats, w0.shape[1], pad
        return D.derived(self, "_dense_mats", [c.weight for c in convs], build)

    def dense_chain(self, context=None):
        """dense.ConvChain describing this net on PIXEL ROWS ([B*H*W, C], channels last), or None when it needs the torch path:
        only inside a native image chain (dense.image_geometry set), relu (other activations keep the torch path), no batch norm /
        active dropout / context."""
        from ... import dense as D
        if context is not None or self.context_channels is not None or D.current_geometry() is None or D.backend() != "tc":
            return None
        for block in self.blocks:
            if (block.use_batch_norm or D.activation_code(block.activation) != D.N.ACT_RELU
                    or (block.dropout.p > 0.0 and block.training)):
                return None
            if any(c.kernel_size != (3, 3) or c.padding != (1, 1) or c.stride != (1, 1) for c in block.conv_layers):
                return None
        mats, in_features, pad = self._dense_parts()
        layers = [(mats[0], self.initial_layer.bias, False, False, None)]
        conv = []
        k = 1
        for block in self.blocks:
            c0, c1 = block.conv_layers
            conv += [len(layers), len(layers) + 1]
            layers.append((mats[k], c0.bias, True, True, None))
            layers.append((mats[k + 1], c1.bias, False, False, "skip"))
            k += 2
        layers.append((mats[k], self.final_layer.bias, False, False, None))
        return D.ConvChain(layers, conv, in_features, pad)
