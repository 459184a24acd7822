"""ConvE decoder (Dettmers et al., AAAI 2018; DESIGN.md section 1).

A query (anchor a, relation r, side) becomes a row q = f(codes[a], rho) of the query network: rho = rel[r] for an
object query (s, r, ?) and the reciprocal row rel_inv[r] for a subject query (?, r, o).  f reshapes both rows to
h x w (d = CodeDimension = h w), stacks them into a 2h x w image (anchor on top), applies input dropout, C 3x3 filters
with a bias, ReLU, feature dropout (one bit per query and filter), a fully connected layer W_fc [F, d] + b_fc, hidden
dropout and ReLU.  The energy of candidate v is <q, codes[v]>.  Training is 1-N only (ops.conve_one_to_n_loss); the
regulariser is the L2 of the anchor row and the relation or reciprocal row.  Not built: batch normalisation, the
per-entity output bias and weight decay on the network.  There is no relation prediction (the energy is not linear
in the relation row) and no fused ensemble membership."""
import numpy as np
import torch

from .. import ops
from .bilinear_diag import BilinearDiag

DEFAULT_HEIGHT = 20
DEFAULT_FILTERS = 32
DEFAULT_KEEPS = (('InputDropoutKeepProbability', 0.8), ('FeatureDropoutKeepProbability', 0.8),
                 ('HiddenDropoutKeepProbability', 0.7))


def parse_conve_settings(settings, dimension):
    """(h, C, (input, feature, hidden) keep probabilities) of [Decoder]: EmbeddingHeight h (default 20) with
    CodeDimension = h w, h >= 2, w >= 3 and CodeDimension % 4 == 0; ConvFilters C >= 1 (default 32); each keep
    probability in (0, 1] (defaults 0.8 / 0.8 / 0.7)."""
    h = int(settings['EmbeddingHeight']) if 'EmbeddingHeight' in settings else DEFAULT_HEIGHT
    if dimension % 4:
        raise ValueError("the ConvE decoder needs CodeDimension %% 4 == 0, got %d" % dimension)
    if h < 2 or dimension % h or dimension // h < 3:
        raise ValueError("the ConvE decoder needs CodeDimension = EmbeddingHeight * w with EmbeddingHeight >= 2 and "
                         "w >= 3, got CodeDimension %d and EmbeddingHeight %d" % (dimension, h))
    C = int(settings['ConvFilters']) if 'ConvFilters' in settings else DEFAULT_FILTERS
    if C < 1:
        raise ValueError("ConvFilters must be >= 1, got %d" % C)
    keeps = []
    for key, default in DEFAULT_KEEPS:
        k = float(settings[key]) if key in settings else default
        if not 0.0 < k <= 1.0:
            raise ValueError("%s must be in (0, 1], got %r" % (key, k))
        keeps.append(k)
    return h, C, tuple(keeps)


def _glorot(rows, cols, fan_in, fan_out):
    limit = np.sqrt(6.0 / (fan_in + fan_out))
    return np.random.uniform(-limit, limit, size=(rows, cols)).astype(np.float32)


class ConvE(BilinearDiag):
    ONE_TO_N = "conve"
    # query rows from a network: the ensemble's fused kernel combines the shallow decoders only
    ensemble_fused = False

    def __init__(self, dimension, settings, next_component=None):
        self.dimension = dimension
        BilinearDiag.__init__(self, next_component, settings)

    def parse_settings(self):
        BilinearDiag.parse_settings(self)
        self.height, self.filter_count, self.keeps = parse_conve_settings(self.settings, self.dimension)

    @property
    def feature_count(self):
        h, w = self.height, self.dimension // self.height
        return self.filter_count * (2 * h - 2) * (w - 2)

    def local_initialize_train(self):
        BilinearDiag.local_initialize_train(self)
        d, C, F, R = self.dimension, self.filter_count, self.feature_count, self.relation_count
        dev = self.get_device()
        # the reciprocal rows as the encoders' relation table (standard normal, numpy's global stream); the network
        # Glorot-uniform with zero biases
        self.W_relation_inverse = torch.from_numpy(np.random.randn(R, d).astype(np.float32)).to(dev)
        self.W_relation_inverse.requires_grad_(True)
        self.W_filters = torch.from_numpy(_glorot(C, 9, 9, 9 * C).reshape(C, 3, 3)).to(dev).requires_grad_(True)
        self.b_conv = torch.zeros(C, dtype=torch.float32, device=dev, requires_grad=True)
        self.W_fc = torch.from_numpy(_glorot(F, d, F, d)).to(dev).requires_grad_(True)
        self.b_fc = torch.zeros(d, dtype=torch.float32, device=dev, requires_grad=True)

    def local_get_weights(self):
        return [self.W_relation_inverse, self.W_filters, self.b_conv, self.W_fc, self.b_fc]

    def network(self):
        """ops.ConvEWeights of the decoder's own weights."""
        return ops.ConvEWeights(self.W_relation_inverse, self.W_filters, self.b_conv, self.W_fc, self.b_fc,
                                self.height)

    def _drop_masks(self, n):
        """The (input, feature, hidden) keep-masks of n training queries, drawn on the device; None where keep = 1."""
        dev = self.get_device()
        widths = (2 * self.dimension, self.filter_count, self.dimension)
        return tuple(None if k >= 1.0 else (torch.rand(n, w, device=dev) < k).to(torch.uint8)
                     for k, w in zip(self.keeps, widths))

    def _one_to_n_op(self, codes, rel, queries, labels):
        return ops.conve_one_to_n_loss(codes, rel, self.network(), queries, labels, self.label_smoothing,
                                       self._drop_masks(len(queries)), self.keeps, self.relation_count)

    def _score_op(self):
        raise NotImplementedError("the ConvE decoder scores queries against every entity: it trains under "
                                  "TrainingObjective=1-N only")

    def _ranker(self, codes, rel):
        return ops.ConvERanker(codes, rel, self.network(), self.relation_count)

    def _query_rows(self, side):
        """Test-mode query rows of the fed triples: side 1 f(e_s, rel[r]), side 0 f(e_o, rel_inv[r])."""
        subject_codes, relation_codes, _ = self.next_component.get_all_codes(mode='test')
        return ops.conve_query_rows(subject_codes.contiguous(), relation_codes.contiguous(), self.network(),
                                    self._x_device(), side, self.relation_count)

    def predict(self):
        """float32 sigmoid(f(e_s, rel[r]) . e_o) of the fed triples."""
        codes = self.next_component.get_all_codes(mode='test')[0]
        X = self._x_device().long()
        return torch.sigmoid((self._query_rows(1) * codes[X[:, 2]]).sum(1))

    def predict_all_subject_scores(self):
        """[n, V]: every entity as the subject, q = f(e_o, rel_inv[r])."""
        all_subject_codes = self.next_component.get_all_subject_codes(mode='test')
        return torch.sigmoid(self._query_rows(0) @ all_subject_codes.T)

    def predict_all_object_scores(self):
        """[n, V]: every entity as the object, q = f(e_s, rel[r])."""
        all_object_codes = self.next_component.get_all_object_codes(mode='test')
        return torch.sigmoid(self._query_rows(1) @ all_object_codes.T)
