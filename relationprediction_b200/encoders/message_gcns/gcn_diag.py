"""DiagGcn: R-GCN layer with one diagonal weight per relation and direction, selected by Encoder Name=gcn_diag
(reference: encoders/message_gcns/gcn_diag.py).  A message s -> o of relation r is D_forward[r] * H[s] (element-wise;
the backward message o -> s is D_backward[r] * H[o]); unlike BasisGcn and ConcatGcn the bias b is added.

The reference spells the element-wise product `tf.mul` (:35-36), which TensorFlow removed in 1.0, so the reference
raises AttributeError when it builds this layer; the port computes the product the name stands for (tf.multiply)."""
from ...common.shared_functions import glorot_variance, make_variable, make_bias
from ... import ops
from .message_gcn import MessageGcn


class DiagGcn(MessageGcn):
    def __init__(self, shape, settings, next_component=None, onehot_input=False, use_nonlinearity=True):
        if onehot_input:
            raise NotImplementedError("DiagGcn reads feature input only: the reference's gcn_diag encoder always "
                                      "puts an input AffineTransform in front of it (model_builder.py:89-94)")
        MessageGcn.__init__(self, shape, settings, next_component, onehot_input, use_nonlinearity)

    def parse_settings(self):
        self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])

    def local_initialize_train(self):
        dev = self.get_device()
        type_matrix_shape = (self.relation_count, self.shape[1])                            # :14
        self.W_self = make_variable(0, glorot_variance(self.shape), tuple(self.shape), dev)  # :17-18
        self.D_types_forward = make_variable(0, 1, type_matrix_shape, dev)                   # :20-22, std 1
        self.D_types_backward = make_variable(0, 1, type_matrix_shape, dev)
        self.b = make_bias(self.shape[1], dev)                                               # :24

    def local_get_weights(self):
        return [self.D_types_forward, self.D_types_backward, self.W_self, self.b]

    def fused_layer(self, H, graph, mode):
        mask, keep = self.make_drop_mask(graph.handle.V_dst, mode)
        return ops.diag_layer(H, self.D_types_forward, self.D_types_backward, self.W_self, self.b, graph.handle,
                              mask, keep, self.use_nonlinearity)

    def local_get_regularization(self):
        return 0.0   # the reference layer defines no local_get_regularization
