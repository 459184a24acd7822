"""Model base class: the reference's plugin protocol (code/model.py:8-182) with TensorFlow removed.

A model is a linked list of components (`next_component`); calls either delegate down the chain
(`__delegate__`), run locally then delegate (`__local_run_delegate__`), or concatenate local results
after the deeper component's (`__local_expand_delegate__`: deepest component first, model.py:179-182).
Where the reference built a TF graph and executed it with session.run, components here execute
eagerly: placeholders are `Placeholder` holders the caller feeds, weights are torch CUDA tensors, and
the hot ops are single calls into librgcn_b200.so (relationprediction_b200/ops.py).
"""
import numpy as np
import torch


class Placeholder(object):
    """Stand-in for tf.placeholder: a named slot the driver feeds before a run (model.py:51-56)."""

    def __init__(self, name, dtype, shape):
        self.name, self.dtype, self.shape = name, dtype, shape
        self.value = None
        self.version = 0

    def set(self, value):
        self.value = value
        self.version += 1

    def __repr__(self):
        return "<Placeholder %s %s %s>" % (self.name, self.dtype, self.shape)


class Model(object):
    next_component = None
    save_iter = 0
    device = None

    def __init__(self, next_component, settings):
        self.next_component = next_component
        self.settings = settings
        self.entity_count = int(self.settings['EntityCount'])
        self.relation_count = int(self.settings['RelationCount'])
        self.edge_count = int(self.settings['EdgeCount'])
        self.parse_settings()

    def parse_settings(self):
        pass

    # ---- device plumbing (the reference had one implicit tf.Session) ----
    def get_device(self):
        if self.device is not None:
            return self.device
        if self.next_component is not None:
            return self.next_component.get_device()
        return torch.device("cuda", torch.cuda.current_device())

    def set_device(self, device):
        self.device = torch.device(device)
        if self.next_component is not None:
            self.next_component.set_device(device)

    # ---- checkpoint (model.py:30-39: Saver over get_weights(), global_step = save_iter) ----
    def save(self, save_path):
        print("saving...")
        torch.save([w.detach().cpu() for w in self.get_weights()], "%s-%d.pt" % (save_path, self.save_iter))
        self.save_iter += 1

    def load(self, path):
        for w, v in zip(self.get_weights(), torch.load(path)):
            with torch.no_grad():
                w.copy_(v.to(w.device))

    # ---- high-level scoring (model.py:46-81) ----
    def _feed_test(self, graph_triplets, triplets):
        inputs = self.get_test_input_variables()
        if self.needs_graph():
            inputs[0].set(np.asarray(graph_triplets))
            inputs[1].set(np.asarray(triplets))
        else:
            inputs[0].set(np.asarray(triplets))
        self.clear_cache()

    def score(self, triplets):
        self._feed_test(getattr(self, 'train_triplets', None), triplets)
        with torch.no_grad():
            return self.predict().cpu().numpy()

    def score_all_subjects(self, triplets):
        self._feed_test(getattr(self, 'test_graph', None), triplets)
        with torch.no_grad():
            return self.predict_all_subject_scores().cpu().numpy()

    def score_all_objects(self, triplets):
        self._feed_test(getattr(self, 'test_graph', None), triplets)
        with torch.no_grad():
            return self.predict_all_object_scores().cpu().numpy()

    def supports_fused_ranking(self):
        """True when the head decoder has a fused scorer/ranker and the model lives on a CUDA device."""
        return hasattr(self, 'rank_all') and self.get_device().type == 'cuda'

    def rank_all_entities(self, triplets, known_subject_lists, known_object_lists):
        """Ranks under both corruptions through the decoder's fused scorer/ranker (one encoder pass for the whole
        set); decoders without one return None and the Scorer falls back to score_all_subjects / score_all_objects."""
        if not hasattr(self, 'rank_all'):
            return None
        self._feed_test(getattr(self, 'test_graph', None), np.asarray(triplets).reshape(-1, 3)[:1])
        with torch.no_grad():
            return self.rank_all(triplets, known_subject_lists, known_object_lists)

    def entity_ranker(self, triplets):
        """The head decoder's fused ranker over the test codes (ops.DistMultRanker / ops.ComplexRanker), fed like
        rank_all_entities: one encoder pass in test mode.  None for decoders without one or off CUDA."""
        if not self.supports_fused_ranking() or not hasattr(self, 'test_ranker'):
            return None
        self._feed_test(getattr(self, 'test_graph', None), np.asarray(triplets).reshape(-1, 3)[:1])
        with torch.no_grad():
            return self.test_ranker()

    def predict_top_k(self, triplets, k, side, exclude_lists=None):
        """The k most likely entities for every triple under the decoder's fused top-k path (one encoder pass for
        the whole set), fed like rank_all_entities.  side 0 predicts subjects, 1 objects; the predicted column of
        `triplets` is not read but must hold an entity id.  exclude_lists[t] (optional) lists the entities row t
        may not return.  Returns numpy (ids [n, k], energies [n, k], scores = float32 sigmoid(energies)); rows with
        fewer than k eligible entities end in id -1, energy -inf, score 0."""
        if not hasattr(self, 'top_k_all') or self.get_device().type != 'cuda':
            raise NotImplementedError("%s has no fused top-k prediction on a CUDA device (DistMult and ComplEx "
                                      "decoders on CUDA have one)" % type(self).__name__)
        k, side = int(k), int(side)
        if side not in (0, 1):
            raise ValueError("side must be 0 (predict subjects) or 1 (predict objects), got %r" % (side,))
        if not 1 <= k <= 128:
            raise ValueError("k must be in [1, 128], got %d" % k)
        triplets = np.asarray(triplets).reshape(-1, 3)
        self._feed_test(getattr(self, 'test_graph', None), triplets[:1])
        with torch.no_grad():
            ids, energies = self.top_k_all(triplets, k, side, exclude_lists)
        with np.errstate(over='ignore'):   # exp(+inf) of the padding: score 0
            scores = (1.0 / (1.0 + np.exp(-energies.astype(np.float32)))).astype(np.float32)
        return ids, energies, scores

    def _relation_triplets(self, hook, triplets, check_relations):
        if not hasattr(self, hook) or self.get_device().type != 'cuda':
            raise NotImplementedError("%s has no fused relation prediction on a CUDA device (DistMult and ComplEx "
                                      "decoders on CUDA have one)" % type(self).__name__)
        triplets = np.asarray(triplets).reshape(-1, 3)
        if len(triplets):
            ent = triplets[:, [0, 2]]
            if ent.min() < 0 or ent.max() >= self.entity_count:
                raise ValueError("entity ids must be in [0, %d)" % self.entity_count)
            if check_relations and (triplets[:, 1].min() < 0 or triplets[:, 1].max() >= self.relation_count):
                raise ValueError("relation ids must be in [0, %d)" % self.relation_count)
        self._feed_test(getattr(self, 'test_graph', None), triplets[:1])
        return triplets

    def rank_all_relations(self, triplets, known_relation_lists):
        """Ranks of every triple's relation among the RelationCount relations for its (head, tail) pair, through the
        decoder's fused relation ranker (one encoder pass for the whole set), fed like rank_all_entities.
        known_relation_lists[t] lists the relations r with (head, r, tail) known; the filtered rank leaves them out
        as the entity ranks do.  Returns numpy (raw, filtered) int64 [n]."""
        triplets = self._relation_triplets('rank_relations_all', triplets, check_relations=True)
        with torch.no_grad():
            return self.rank_relations_all(triplets, known_relation_lists)

    def predict_top_k_relations(self, triplets, k, exclude_lists=None):
        """The k most likely relations for every (head, ?, tail) pair of `triplets` (the relation column is not
        read) under the decoder's fused path, fed like predict_top_k.  exclude_lists[t] (optional) lists the
        relations row t may not return.  Returns numpy (ids [n, k], energies [n, k], scores = float32
        sigmoid(energies)); rows with fewer than k eligible relations end in id -1, energy -inf, score 0."""
        k = int(k)
        if not 1 <= k <= 128:
            raise ValueError("k must be in [1, 128], got %d" % k)
        triplets = self._relation_triplets('top_k_relations_all', triplets, check_relations=False)
        with torch.no_grad():
            ids, energies = self.top_k_relations_all(triplets, k, exclude_lists)
        with np.errstate(over='ignore'):   # exp(+inf) of the padding: score 0
            scores = (1.0 / (1.0 + np.exp(-energies.astype(np.float32)))).astype(np.float32)
        return ids, energies, scores

    def register_for_test(self, triplets):
        self.test_graph = triplets

    def preprocess(self, triplets):
        self.train_triplets = triplets

    # ---- one eager training evaluation: feed [graph_edges, X, Y] (train.py:245) -> scalar loss ----
    def train_loss(self, *feed):
        for ph, value in zip(self.get_train_input_variables(), feed):
            ph.set(value)
        self.clear_cache()
        return self.get_loss(mode='train') + self.get_regularization()

    def needs_graph(self):
        nxt = self.next_component
        return False if nxt is None else nxt.needs_graph()

    # ---- the three call disciplines of the chain (code/model.py:148-182) ----
    def __delegate__(self, name, *args, **kw):
        """Pure forwarding to the next component; None at the end of the chain."""
        nxt = self.next_component
        return None if nxt is None else getattr(nxt, name)(*args, **kw)

    def __local_run_delegate__(self, name, *args, **kw):
        """Run `local_<name>` here if this component defines it, then continue down the chain."""
        hook = getattr(self, 'local_' + name, None)
        if hook is not None:
            hook(*args, **kw)
        if self.next_component is not None:
            getattr(self.next_component, name)(*args, **kw)

    def __local_expand_delegate__(self, name, *args, base=None, **kw):
        """Collect `local_<name>` results along the chain, DEEPEST component first (this fixes the order
        of get_weights() and of the feed lists)."""
        hook = getattr(self, 'local_' + name, None)
        mine = hook(*args, **kw) if hook is not None else ([] if base is None else base)
        if self.next_component is None:
            return mine
        return getattr(self.next_component, name)(*args, **kw) + mine


def _install_chain_protocol(cls):
    """The public hooks of the plugin protocol, generated from one table: which discipline each follows."""
    def forward(name):
        return lambda self, *a, **k: self.__delegate__(name, *a, **k)

    def run(name):
        return lambda self, *a, **k: self.__local_run_delegate__(name, *a, **k)

    def collect(name, base):
        return lambda self, *a, **k: self.__local_expand_delegate__(name, *a, base=base, **k)
    table = {
        forward: ('get_loss', 'get_all_subject_codes', 'get_all_object_codes', 'get_all_codes', 'predict',
                  'predict_all_subject_scores', 'predict_all_object_scores', 'get_graph'),
        run: ('initialize_train', 'clear_cache', 'set_variable'),
    }
    for make, names in table.items():
        for name in names:
            fn = make(name)
            fn.__name__ = name
            setattr(cls, name, fn)
    for name, base in (('get_weights', None), ('get_train_input_variables', None),
                       ('get_test_input_variables', None), ('get_additional_ops', None),
                       ('get_regularization', 0)):
        fn = collect(name, base)
        fn.__name__ = name
        setattr(cls, name, fn)


_install_chain_protocol(Model)
