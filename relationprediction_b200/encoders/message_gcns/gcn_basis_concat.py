"""ConcatGcn: block-diagonal R-GCN layer (reference: encoders/message_gcns/gcn_basis_concat.py)."""
from ...common.shared_functions import glorot_variance, make_variable, make_bias
from ... import ops
from .message_gcn import MessageGcn


class ConcatGcn(MessageGcn):
    def __init__(self, shape, settings, next_component=None, onehot_input=False, use_nonlinearity=True):
        if onehot_input:
            raise NotImplementedError(
                "ConcatGcn has no one-hot input layer: the reference reshapes the integer index vector as "
                "[-1, B, s] features (gcn_basis_concat.py:42-43) and cannot run with UseInputTransform=No")
        MessageGcn.__init__(self, shape, settings, next_component, onehot_input, use_nonlinearity)

    def parse_settings(self):
        self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])
        self.n_coefficients = int(self.settings['NumberOfBasisFunctions'])
        self.submatrix_d = int(self.shape[1] / self.n_coefficients)

    def local_initialize_train(self):
        dev = self.get_device()
        vertex_matrix_shape = (self.relation_count, self.n_coefficients, self.submatrix_d, self.submatrix_d)
        std = glorot_variance([vertex_matrix_shape[0], vertex_matrix_shape[2]])  # gcn_basis_concat.py:22
        self.W_forward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_backward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_self = make_variable(0, std, tuple(self.shape), dev)
        self.b = make_bias(self.shape[1], dev)  # listed as a weight, never added (reference behaviour)

    def local_get_weights(self):
        return [self.W_forward, self.W_backward, self.W_self, self.b]

    def fused_layer(self, H, graph, mode):
        mask, keep = self.make_drop_mask(graph.handle.V_dst, mode)
        return ops.block_layer(H, self.W_forward, self.W_backward, self.W_self, graph.handle,
                               self.n_coefficients, mask, keep, self.use_nonlinearity)

    def local_get_regularization(self):
        return 0.0  # 0.0 * (...) in the reference (gcn_basis_concat.py:85-90)
