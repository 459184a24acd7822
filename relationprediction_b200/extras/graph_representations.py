"""Graph representation plugin (reference: extras/graph_representations.py).

`Representation` owns the int32 [E,3] edge placeholder (:173-174); `MessageGraph` exposes the index
vectors (:21-27) and the per-direction normalisation values (:84-93, :124-133) and, new here, the
prepared device graph handle (ops.Graph) every layer shares.  The incidence matrices themselves are
never materialised: their VALUES are the per-message `norm` array of the handle."""
import numpy as np
import torch

from ..model import Model, Placeholder
from .. import ops


class MessageGraph(object):
    def __init__(self, edges, vertex_count, label_count, device, norm_mode="canonical",
                 norm_f=None, norm_b=None):
        self.vertex_count = vertex_count
        self.label_count = label_count
        self.edges = np.ascontiguousarray(np.asarray(edges, dtype=np.int32).reshape(-1, 3))
        self.device = device
        self.process(self.edges)
        index = device.index if device.index is not None else torch.cuda.current_device()
        self.handle = ops.Graph(self.edges, vertex_count, label_count, norm_mode=norm_mode,
                                norm_f=norm_f, norm_b=norm_b, device=index)

    def process(self, triplets):
        self.sender_indices = triplets[:, 0]
        self.receiver_indices = triplets[:, 2]
        self.message_types = triplets[:, 1]
        self.edge_count = triplets.shape[0]

    def get_sender_indices(self):
        return self.sender_indices

    def get_type_indices(self):
        return self.message_types

    def get_receiver_indices(self):
        return self.receiver_indices

    def _values(self, which):
        from .. import _lib
        norm = self.handle.export(_lib.X_MSG_NORM)
        E = self.edge_count
        return norm[:E] if which == 'forward' else norm[E:]

    def forward_incidence_matrix(self, normalization):
        """(row indices = receivers, column = message id, values) of the [V,E] incidence (:69-93)."""
        vals = np.ones(self.edge_count, np.float32) if normalization[0] == "none" else self._values('forward')
        return self.receiver_indices, np.arange(self.edge_count), vals

    def backward_incidence_matrix(self, normalization):
        vals = np.ones(self.edge_count, np.float32) if normalization[0] == "none" else self._values('backward')
        return self.sender_indices, np.arange(self.edge_count), vals


class Representation(Model):
    normalization = "global"
    norm_mode = "canonical"   # or "tf_unsorted_compat" (quirk Q1, see DESIGN.md), or "relation" (the 'local' branch)

    def __init__(self, triples, settings, bipartite=False):
        self.settings = settings
        self.next_component = None
        self.triples = np.array(triples)
        self.entity_count = int(settings['EntityCount'])
        self.relation_count = int(settings['RelationCount'])
        self.edge_count = self.triples.shape[0] * 2
        self.X = None
        self._graphs = {}
        if 'NormalizationMode' in settings:
            self.norm_mode = settings['NormalizationMode']

    def needs_graph(self):
        return True

    def local_initialize_train(self):
        self.X = Placeholder('graph_edges', 'int32', [None, 3])

    def local_get_train_input_variables(self):
        return [self.X]

    def local_get_test_input_variables(self):
        return [self.X]

    def local_get_weights(self):
        return []

    def get_graph(self):
        """The prepared graph of the currently fed edge list; handles are cached by content so the
        evaluation loop, which feeds the same training graph for every chunk (model.py:59-81), pays
        for graph preparation once."""
        edges = np.ascontiguousarray(np.asarray(self.X.value, dtype=np.int32).reshape(-1, 3))
        key = (edges.shape[0], hash(edges.tobytes()))
        g = self._graphs.get(key)
        if g is None:
            if len(self._graphs) >= 4:
                self._graphs.pop(next(iter(self._graphs)))
            kw = {}
            if self.norm_mode == "tf_unsorted_compat":
                kw = dict(norm_mode="explicit", norm_f=_tf_compat(edges[:, 2], self.entity_count),
                          norm_b=_tf_compat(edges[:, 0], self.entity_count))
            elif self.norm_mode == "relation":
                # per-relation c_{i,r}: the 'local' branch of the incidence matrices (:94-107, :134-147)
                kw = dict(norm_mode="relation")
            g = MessageGraph(edges, self.entity_count, self.relation_count, self.get_device(), **kw)
            self._graphs[key] = g
        return g


def _tf_compat(rows, n):
    """Quirk Q1: values computed in canonical (sorted) order, re-attached to the unsorted entries."""
    rows = np.asarray(rows, dtype=np.int64)
    counts = np.bincount(rows, minlength=n).astype(np.float32)
    order = np.argsort(rows, kind="stable")
    return (np.float32(1.0) / counts[rows[order]]).astype(np.float32)
