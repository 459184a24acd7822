"""BasisGcn: basis-decomposition R-GCN layer (reference: encoders/message_gcns/gcn_basis.py)."""
from ...common.shared_functions import glorot_variance, make_variable, make_bias
from ... import ops
from .message_gcn import MessageGcn


class BasisGcn(MessageGcn):
    def parse_settings(self):
        self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])
        self.n_coefficients = int(self.settings['NumberOfBasisFunctions'])

    def local_initialize_train(self):
        dev = self.get_device()
        d_in = self.entity_count if self.onehot_input else self.shape[0]   # gcn_basis.py:16
        type_matrix_shape = (self.relation_count, self.n_coefficients)
        vertex_matrix_shape = (d_in, self.n_coefficients, self.shape[1])
        std = glorot_variance([vertex_matrix_shape[0], vertex_matrix_shape[2]])  # gcn_basis.py:21
        self.W_forward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_backward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_self = make_variable(0, std, (d_in, self.shape[1]), dev)
        self.C_forward = make_variable(0, 1, type_matrix_shape, dev)            # gcn_basis.py:26-28
        self.C_backward = make_variable(0, 1, type_matrix_shape, dev)
        self.b = make_bias(self.shape[1], dev)

    def local_get_weights(self):
        return [self.W_forward, self.W_backward, self.C_forward, self.C_backward, self.W_self, self.b]

    def fused_layer(self, H, graph, mode):
        mask, keep = self.make_drop_mask(graph.handle.V_dst, mode)
        if self.onehot_input:
            return ops.basis_onehot_layer(self.W_forward, self.W_backward, self.C_forward, self.C_backward,
                                          self.W_self, graph.handle, mask, keep, self.use_nonlinearity)
        return ops.basis_layer(H, self.W_forward, self.W_backward, self.C_forward, self.C_backward,
                               self.W_self, graph.handle, mask, keep, self.use_nonlinearity)

    def local_get_regularization(self):
        return 0.0
