"""BasisGcnTimesDiag: basis R-GCN layer with per-channel sigmoid coefficients, selected by DiagonalCoefficients=Yes
(reference: encoders/message_gcns/gcn_basis_times_diag.py).  A message s -> o of relation r is
sum_b sigmoid(C_dir[r, b, :]) * (H[s] @ W_dir[:, b, :]); unlike BasisGcn and ConcatGcn the bias b is added."""
from ...common.shared_functions import glorot_variance, make_variable, make_bias
from ... import ops
from .message_gcn import MessageGcn


class BasisGcnTimesDiag(MessageGcn):
    def __init__(self, shape, settings, next_component=None, onehot_input=False, use_nonlinearity=True):
        if onehot_input:
            raise NotImplementedError(
                "DiagonalCoefficients=Yes with UseInputTransform=No: the featureless first layer would need its own "
                "per-channel push kernel over the [V, B, d] tables, which is not built")
        MessageGcn.__init__(self, shape, settings, next_component, onehot_input, use_nonlinearity)

    def parse_settings(self):
        self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])
        self.n_coefficients = int(self.settings['NumberOfBasisFunctions'])

    def local_initialize_train(self):
        dev = self.get_device()
        type_matrix_shape = (self.relation_count, self.n_coefficients, self.shape[1])     # :22
        vertex_matrix_shape = (self.shape[0], self.n_coefficients, self.shape[1])
        std = glorot_variance([vertex_matrix_shape[0], vertex_matrix_shape[2]])          # :26
        self.W_forward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_backward = make_variable(0, std, vertex_matrix_shape, dev)
        self.W_self = make_variable(0, std, (self.shape[0], self.shape[1]), dev)
        self.C_forward = make_variable(0, 1, type_matrix_shape, dev)                      # :31-33
        self.C_backward = make_variable(0, 1, type_matrix_shape, dev)
        self.b = make_bias(self.shape[1], dev)

    def local_get_weights(self):
        return [self.W_forward, self.W_backward, self.C_forward, self.C_backward, self.W_self, self.b]

    def fused_layer(self, H, graph, mode):
        mask, keep = self.make_drop_mask(graph.handle.V_dst, mode)
        return ops.basis_diagcoef_layer(H, self.W_forward, self.W_backward, self.C_forward, self.C_backward,
                                        self.W_self, self.b, graph.handle, mask, keep, self.use_nonlinearity)

    def local_get_regularization(self):
        return 0.0   # the reference layer defines no local_get_regularization
