"""HighwayLayer: gated skip connection around one R-GCN layer (reference: extras/highway_layer.py, wired by
model_builder.py:304-305 when SkipConnections=Highway).

  out = g * c1 + (1 - g) * c2,   g = sigmoid(c2 @ W + b)

c1 is the wrapped layer's output (`next_component`), c2 the layer's input (`next_component_2`: the previous highway's
output, or the input transform below layer 0).  The gate GEMM, sigmoid and blend are one library call (ops.highway).
Memoisation is per INSTANCE and dropped by Model.clear_cache(), like MessageGcn here; the reference's class-level
dict gives the same result whenever the first layer reads features (UseInputTransform=Yes), which is the only
configuration model_builder wraps."""
from ..common.shared_functions import glorot_variance, make_variable, make_bias
from ..model import Model
from .. import ops


class HighwayLayer(Model):
    def __init__(self, shape, next_component=None, next_component_2=None):
        self.next_component = next_component
        self.next_component_2 = next_component_2
        self.shape = shape
        self.vertex_embedding_function = {'train': None, 'test': None}

    def local_initialize_train(self):
        dev = self.get_device()
        self.W = make_variable(0, glorot_variance(self.shape), self.shape, dev)   # highway_layer.py:26-28
        self.b = make_bias(self.shape[1], dev, init=1)                          # :29, make_tf_bias(init=1)

    def local_get_weights(self):
        return [self.W, self.b]

    def local_clear_cache(self):
        self.vertex_embedding_function = {'train': None, 'test': None}

    def compute_vertex_embeddings(self, mode='train'):
        if self.vertex_embedding_function[mode] is None:
            code_1 = self.next_component.get_all_codes(mode=mode)[0].contiguous()
            code_2 = self.next_component_2.get_all_codes(mode=mode)[0].contiguous()
            self.vertex_embedding_function[mode] = ops.highway(code_1, code_2, self.W, self.b)
        return self.vertex_embedding_function[mode]

    def get_all_codes(self, mode='train'):
        collected = self.compute_vertex_embeddings(mode=mode)
        return collected, None, collected

    def get_all_subject_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)

    def get_all_object_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)
