"""CompGcn: composition message passing (Vashishth et al., ICLR 2020), selected by Encoder Name=compgcn.

A message s -> o of relation r is phi(H[s], Z[r]) (its inverse o -> s: phi(H[o], Z[R + r])) with phi = h * z
(Composition=mult, the default) or h - z (Composition=sub).  Each layer

    out    = act([M * [A_f | A_b] / keep | phi(H, z_loop)] / 3 @ W_cat + b),     W_cat = [W_I; W_O; W_S]
    Z_next = Z @ W_rel

learns the relation table together with the entity codes: the bottom layer owns Z^0 [2R, d_0], every layer reads Z
from the slot below and hands Z_next up in the relation slot of get_all_codes, and the top layer hands the decoder
Z^L[0:R], a contiguous [R, CodeDimension] tensor.  A_f / A_b are the two directions' normalised message sums (the
graph's norm, NormalizationMode applies), M the train-mode dropout mask on those two slabs, act ReLU except on the
last layer.  Differences from the paper's code: the graph's norm instead of 1/sqrt(deg deg), ReLU instead of tanh,
no batch norm, the dropout on the message slabs before W_I / W_O, no basis-decomposed relation initialisation and
no circular correlation (Composition=corr raises NotImplementedError)."""
import torch

from ...common.shared_functions import glorot_variance, make_variable, make_bias
from ... import ops
from .message_gcn import MessageGcn

COMPOSITIONS = ops.COMPOSITIONS


def parse_composition(settings):
    """Composition of [Encoder]: 'mult' (the default) or 'sub'."""
    composition = str(settings['Composition']) if 'Composition' in settings else 'mult'
    if composition == 'corr':
        raise NotImplementedError("Composition=corr (circular correlation) is not built: use mult or sub")
    if composition not in COMPOSITIONS:
        raise ValueError("Composition must be one of %s, got %r" % (", ".join(COMPOSITIONS), composition))
    return composition


class CompGcn(MessageGcn):
    """One CompGCN layer of shape [d_in, d_out].  owns_relations: the bottom layer, which holds Z^0;
    top: the last layer, which hands Z^L[0:R] to the decoder."""

    def __init__(self, shape, settings, next_component=None, use_nonlinearity=True, owns_relations=False,
                 top=False):
        self.owns_relations = owns_relations
        self.top = top
        MessageGcn.__init__(self, shape, settings, next_component, onehot_input=False,
                            use_nonlinearity=use_nonlinearity)

    def parse_settings(self):
        self.dropout_keep_probability = float(self.settings['DropoutKeepProbability'])
        self.composition = parse_composition(self.settings)

    def local_initialize_train(self):
        dev = self.get_device()
        d_in, d_out = self.shape
        if self.owns_relations:
            relation_shape = (2 * self.relation_count, d_in)
            self.Z = make_variable(0, glorot_variance(relation_shape), relation_shape, dev)
        self.z_loop = make_variable(0, glorot_variance((1, d_in)), (d_in,), dev)
        self.W_cat = make_variable(0, glorot_variance((3 * d_in, d_out)), (3 * d_in, d_out), dev)
        self.W_rel = make_variable(0, glorot_variance((d_in, d_out)), (d_in, d_out), dev)
        self.b = make_bias(d_out, dev)

    def local_get_weights(self):
        return ([self.Z] if self.owns_relations else []) + [self.z_loop, self.W_cat, self.W_rel, self.b]

    def make_drop_mask(self, rows, mode):
        """The keep-mask of the two message slabs [A_f | A_b], train mode only."""
        if mode != 'train' or self.dropout_keep_probability >= 1.0:
            return None, 1.0
        mask = (torch.rand(rows, 2 * self.shape[0], device=self.get_device())
                < self.dropout_keep_probability).to(torch.uint8)
        return mask, self.dropout_keep_probability

    def fused_layer(self, H, graph, mode):
        Z = self.Z if self.owns_relations else self.next_component.get_all_codes(mode=mode)[1].contiguous()
        mask, keep = self.make_drop_mask(graph.handle.V_dst, mode)
        return ops.compgcn_layer(H, Z, self.z_loop, self.W_cat, self.W_rel, self.b, graph.handle, self.composition,
                                 mask, keep, self.use_nonlinearity)

    def get_all_codes(self, mode='train'):
        out, Z_next = self.compute_vertex_embeddings(mode=mode)
        return out, (Z_next[:self.relation_count] if self.top else Z_next), out

    def get_all_subject_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)[0]

    def get_all_object_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)[0]

    def local_get_regularization(self):
        return 0.0
