"""VariationalEncoding: reparameterised entity codes (reference: extras/variational_encoding.py, wired by
model_builder.py:43-69 and :186-254).

  z = mu + exp(l) * eps,   eps ~ N(0, 1) of shape `shape`,   regularisation -0.0005 sum(1 + 2 l - mu^2 - exp(2 l))

mu and l (log sigma) are the outputs of two linear AffineTransform branches: both one-hot (variational_embedding:
mu = W_mu, l = W_sigma) or both reading the same trunk H (variational_gcn_basis: mu = H W_mu + b_mu, l = H W_sigma +
b_sigma).  z and the KL term come from one library call (ops.variational), so the trunk is evaluated once.  eps is
drawn afresh for every evaluation, in train and in test mode, as the reference's tf.random_normal is on every run.
Memoisation is per INSTANCE and dropped by Model.clear_cache(), like MessageGcn here (the reference's class-level
dict is quirk Q5)."""
import torch

from .. import ops
from ..encoders.affine_transform import AffineTransform
from .split_model import SplitModel


class VariationalEncoding(SplitModel):
    def __init__(self, shape, settings, mu_network=None, sigma_network=None):
        branches = (mu_network, sigma_network)
        if not all(isinstance(b, AffineTransform) and not b.use_nonlinearity for b in branches):
            raise NotImplementedError("VariationalEncoding needs two linear AffineTransform branches")
        if mu_network.onehot_input != sigma_network.onehot_input:
            raise NotImplementedError("VariationalEncoding needs both branches one-hot or both on the same trunk")
        if mu_network.onehot_input:
            ok = mu_network.next_component is None and sigma_network.next_component is None \
                and not mu_network.use_bias and not sigma_network.use_bias
        else:
            ok = mu_network.next_component is not None and mu_network.next_component is sigma_network.next_component \
                and mu_network.use_bias and sigma_network.use_bias
        if not ok:
            raise NotImplementedError("VariationalEncoding needs one-hot branches without bias or biased branches "
                                      "over one shared trunk")
        if list(mu_network.shape) != list(sigma_network.shape):
            raise NotImplementedError("VariationalEncoding needs branches of one shape")
        if int(mu_network.shape[1]) != int(shape[1]):
            raise ValueError("the variational code has %d columns but its noise has %d: the reference adds mu "
                             "[EntityCount, CodeDimension] to sigma * eps [EntityCount, InternalEncoderDimension], "
                             "which only broadcasts when CodeDimension == InternalEncoderDimension"
                             % (int(mu_network.shape[1]), int(shape[1])))
        SplitModel.__init__(self, [mu_network, sigma_network], settings)
        self.mu_network = mu_network
        self.sigma_network = sigma_network
        self.shape = shape
        self.vertex_embedding_function = {'train': None, 'test': None}

    def local_clear_cache(self):
        self.vertex_embedding_function = {'train': None, 'test': None}

    def draw_epsilon(self, mode):
        """eps ~ N(0, 1) of shape `shape` on the layer's device, a fresh draw on every evaluation."""
        return torch.randn(int(self.shape[0]), int(self.shape[1]), device=self.get_device())

    def compute_vertex_embeddings(self, mode='train'):
        """(z, KL term) of `mode`."""
        if self.vertex_embedding_function[mode] is None:
            mu, sigma = self.mu_network, self.sigma_network
            H = None if mu.onehot_input else mu.next_component.get_all_codes(mode=mode)[0].contiguous()
            self.vertex_embedding_function[mode] = ops.variational(H, mu.W, mu.b, sigma.W, sigma.b,
                                                                   self.draw_epsilon(mode))
        return self.vertex_embedding_function[mode]

    def local_get_regularization(self):
        return self.compute_vertex_embeddings(mode='train')[1]

    def get_all_codes(self, mode='train'):
        z = self.compute_vertex_embeddings(mode=mode)[0]
        return z, None, z

    def get_all_subject_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)[0]

    def get_all_object_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)[0]
