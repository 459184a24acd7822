"""BilinearDiag = DistMult decoder (reference: decoders/bilinear_diag.py)."""
import numpy as np
import torch

from ..model import Model, Placeholder
from .. import ops


class BilinearDiag(Model):
    def __init__(self, next_component, settings):
        self.encoder_cache = {'train': None, 'test': None}
        self._scored = {'train': None, 'test': None}
        Model.__init__(self, next_component, settings)

    def parse_settings(self):
        self.regularization_parameter = float(self.settings['RegularizationParameter'])

    def local_initialize_train(self):
        self.Y = Placeholder('Y', 'float32', [None])
        self.X = Placeholder('X', 'int32', [None, 3])

    def local_clear_cache(self):
        self.encoder_cache = {'train': None, 'test': None}
        self._scored = {'train': None, 'test': None}

    def local_get_train_input_variables(self):
        return [self.X, self.Y]

    def local_get_test_input_variables(self):
        return [self.X]

    def _x_device(self):
        dev = self.get_device()
        return torch.as_tensor(np.ascontiguousarray(np.asarray(self.X.value, dtype=np.int32).reshape(-1, 3)),
                               device=dev)

    def _fused(self, mode):
        """One fused kernel: three row gathers -> energies (+ sigmoid-CE loss and L2 term in train
        mode).  The gathered e1/r/e2 rows of compute_codes are never materialised."""
        if self._scored[mode] is None:
            subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode=mode)
            assert subject_codes is object_codes, "DistMult kernel expects one shared entity code matrix"
            Y = None
            if mode == 'train':
                Y = torch.as_tensor(np.asarray(self.Y.value, dtype=np.float32), device=self.get_device())
            self._scored[mode] = self._score_op()(subject_codes.contiguous(), relation_codes.contiguous(),
                                                  self._x_device(), Y)
        return self._scored[mode]

    def _score_op(self):
        return ops.distmult

    def _ranker(self, codes, rel):
        return ops.DistMultRanker(codes, rel, self.relation_count)

    def compute_codes(self, mode='train'):
        """(e1s, rs, e2s) row gathers (bilinear_diag.py:14-24) -- only the all-entity scoring GEMMs
        below need them explicitly."""
        if self.encoder_cache[mode] is None:
            subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode=mode)
            X = self._x_device().long()
            self.encoder_cache[mode] = (subject_codes[X[:, 0]], relation_codes[X[:, 1]], object_codes[X[:, 2]])
        return self.encoder_cache[mode]

    def get_loss(self, mode='train'):
        return self._fused(mode)[1]  # reduce_mean(weighted CE, pos_weight forced to 1) (:27-34)

    def local_get_regularization(self):
        return self.regularization_parameter * self._fused('train')[2]  # (:63-69)

    def predict(self):
        return torch.sigmoid(self._fused('test')[0])

    def predict_all_subject_scores(self):
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_subject_codes = self.next_component.get_all_subject_codes(mode='test')
        return torch.sigmoid((all_subject_codes @ (rs * e2s).T).T)

    def predict_all_object_scores(self):
        e1s, rs, e2s = self.compute_codes(mode='test')
        all_object_codes = self.next_component.get_all_object_codes(mode='test')
        return torch.sigmoid((e1s * rs) @ all_object_codes.T)

    # ---- fused all-entity scoring + ranking (next row N3; library entry distmult_rank) ----
    @staticmethod
    def known_bit_mask(lists, n_entities):
        """int32 view of the uint32 [n, ceil(V/32)] bit masks the library expects: bit v of row t = v in lists[t]."""
        words = (n_entities + 31) // 32
        m = np.zeros((len(lists), words), np.uint32)
        lens = np.fromiter((len(l) for l in lists), dtype=np.int64, count=len(lists))
        if lens.sum():
            rows = np.repeat(np.arange(len(lists)), lens)
            cols = np.concatenate([np.asarray(l, dtype=np.int64) for l in lists if len(l)])
            np.bitwise_or.at(m, (rows, cols >> 5), np.left_shift(np.uint32(1), (cols & 31).astype(np.uint32)))
        return m.view(np.int32)

    def rank_all(self, triplets, known_subject_lists, known_object_lists, chunk=4096):
        """Raw and filtered ranks of every triple under subject and object corruption with the rules of
        common/evaluation.py:148-159 / :355-367, without materialising the [n, V] score matrices of
        predict_all_subject_scores / predict_all_object_scores (bilinear_diag.py:51-61): the encoder runs once,
        the scoring GEMM counts `score >= gold` in its epilogue.  Returns four int arrays
        (raw_subjects, filtered_subjects, raw_objects, filtered_objects)."""
        subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode='test')
        assert subject_codes is object_codes, "DistMult ranking expects one shared entity code matrix"
        codes, rel = subject_codes.contiguous(), relation_codes.contiguous()
        ranker = self._ranker(codes, rel)
        V = codes.shape[0]
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        out = [[], [], [], []]
        for c0 in range(0, len(tri), chunk):
            X = torch.as_tensor(tri[c0:c0 + chunk], device=codes.device)
            for side, lists in ((0, known_subject_lists), (1, known_object_lists)):
                mask = torch.as_tensor(self.known_bit_mask(lists[c0:c0 + chunk], V), device=codes.device)
                raw, filt = ranker.rank(X, side, mask)
                out[2 * side].append(raw)
                out[2 * side + 1].append(filt)
        return tuple(torch.cat(o).cpu().numpy().astype(np.int64) if o else np.zeros(0, np.int64) for o in out)

    def top_k_all(self, triplets, k, side, exclude_lists=None, chunk=4096):
        """The k entities of highest energy for every triple (side 0 predicts subjects, 1 objects; the predicted
        column is not read), without the [n, V] score matrices of predict_all_subject_scores /
        predict_all_object_scores (bilinear_diag.py:51-61): the encoder runs once, the codes are split once, and the
        scoring GEMM keeps each row's best k in its epilogue.  exclude_lists[t] lists the entities row t may not
        return (or None: none excluded).  Returns (ids int64 [n, k], energies float32 [n, k]); energy descending,
        the smaller id first on ties; rows with fewer than k eligible entities end in (-1, -inf)."""
        subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode='test')
        assert subject_codes is object_codes, "fused top-k prediction expects one shared entity code matrix"
        codes, rel = subject_codes.contiguous(), relation_codes.contiguous()
        ranker = self._ranker(codes, rel)
        V = codes.shape[0]
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        ids, energies = [], []
        for c0 in range(0, len(tri), chunk):
            X = torch.as_tensor(tri[c0:c0 + chunk], device=codes.device)
            mask = None
            if exclude_lists is not None:
                mask = torch.as_tensor(self.known_bit_mask(exclude_lists[c0:c0 + chunk], V), device=codes.device)
            i, e = ranker.top_k(X, side, k, mask)
            ids.append(i)
            energies.append(e)
        if not ids:
            return np.zeros((0, k), np.int64), np.zeros((0, k), np.float32)
        return torch.cat(ids).cpu().numpy().astype(np.int64), torch.cat(energies).cpu().numpy()

    def test_ranker(self):
        """The decoder's fused ranker (ops.DistMultRanker / ops.ComplexRanker) over the test-mode codes of the fed
        inputs: one encoder pass.  The ensemble ranker (ops.EnsembleRanker) combines two of these."""
        subject_codes, relation_codes, object_codes = self.next_component.get_all_codes(mode='test')
        assert subject_codes is object_codes, "fused ranking expects one shared entity code matrix"
        return self._ranker(subject_codes.contiguous(), relation_codes.contiguous())

    # ---- relation queries (h, ?, t): library entries distmult_relation_rank / distmult_relation_topk ----
    def _relation_ranker(self):
        """The ranker over the test-mode codes, with R = RelationCount relation candidates (rows 0..R-1 of the
        relation table)."""
        return self.test_ranker()

    def rank_relations_all(self, triplets, known_relation_lists, chunk=4096):
        """Raw and filtered ranks of every triple's relation among the RelationCount relations for its (head, tail)
        pair, with the counting rules of rank_all; known_relation_lists[t] lists the relations r with (h, r, t) in
        any split.  One encoder pass, one split of the relation table.  Returns (raw, filtered) int64 arrays."""
        ranker = self._relation_ranker()
        dev = ranker.codes.device
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        raw, filt = [], []
        for c0 in range(0, len(tri), chunk):
            X = torch.as_tensor(tri[c0:c0 + chunk], device=dev)
            mask = torch.as_tensor(self.known_bit_mask(known_relation_lists[c0:c0 + chunk], self.relation_count),
                                   device=dev)
            r, f = ranker.rank_relations(X, mask)
            raw.append(r)
            filt.append(f)
        return tuple(torch.cat(o).cpu().numpy().astype(np.int64) if o else np.zeros(0, np.int64) for o in (raw, filt))

    def top_k_relations_all(self, triplets, k, exclude_lists=None, chunk=4096):
        """The k relations of highest energy for every (head, ?, tail) pair of `triplets` (the relation column is
        not read), among the RelationCount relations.  exclude_lists[t] lists the relations row t may not return (or
        None).  Returns (ids int64 [n, k], energies float32 [n, k]); energy descending, the smaller id first on
        ties; rows with fewer than k eligible relations end in (-1, -inf)."""
        ranker = self._relation_ranker()
        dev = ranker.codes.device
        tri = np.ascontiguousarray(np.asarray(triplets, dtype=np.int32).reshape(-1, 3))
        ids, energies = [], []
        for c0 in range(0, len(tri), chunk):
            X = torch.as_tensor(tri[c0:c0 + chunk], device=dev)
            mask = None
            if exclude_lists is not None:
                mask = torch.as_tensor(self.known_bit_mask(exclude_lists[c0:c0 + chunk], self.relation_count),
                                       device=dev)
            i, e = ranker.top_k_relations(X, k, mask)
            ids.append(i)
            energies.append(e)
        if not ids:
            return np.zeros((0, k), np.int64), np.zeros((0, k), np.float32)
        return torch.cat(ids).cpu().numpy().astype(np.int64), torch.cat(energies).cpu().numpy()
