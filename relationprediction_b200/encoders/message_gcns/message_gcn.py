"""MessageGcn template (reference: encoders/message_gcns/message_gcn.py:9-87).

The reference's template method gathers sender/receiver rows, calls compute_messages /
compute_self_loop_messages / combine_messages and memoises the result per mode.  Here the whole
layer is ONE fused library call (`fused_layer`, implemented by the subclasses): per-edge messages and
per-edge weights are never materialised, so compute_messages/combine_messages do not exist as
separate steps and raise if called.  Memoisation is per INSTANCE (the reference's class-level dict,
quirk Q5, is not reproduced) and is dropped by Model.clear_cache() whenever new inputs are fed."""
import torch

from ...model import Model


class MessageGcn(Model):
    onehot_input = True
    use_nonlinearity = True

    def __init__(self, shape, settings, next_component=None, onehot_input=False, use_nonlinearity=True):
        self.onehot_input = onehot_input
        self.use_nonlinearity = use_nonlinearity
        self.shape = shape
        self.vertex_embedding_function = {'train': None, 'test': None}
        Model.__init__(self, next_component, settings)

    def needs_graph(self):
        return True

    def local_clear_cache(self):
        self.vertex_embedding_function = {'train': None, 'test': None}

    def get_vertex_features(self, senders=True, mode='train'):
        """H[sender] / H[receiver] row gathers (message_gcn.py:28-42) -- kept for API completeness;
        the fused layer gathers rows inside the kernel instead.  One-hot input: the index vector itself."""
        g = self.get_graph()
        idx = g.get_sender_indices() if senders else g.get_receiver_indices()
        if self.onehot_input:
            return idx
        code = self.next_component.get_all_codes(mode=mode)[0]
        return code[torch.as_tensor(idx, device=code.device).long()]

    def make_drop_mask(self, rows, mode):
        """tf.nn.dropout on the self-loop messages, train mode only (message_gcn.py:60-64)."""
        if mode != 'train' or self.dropout_keep_probability >= 1.0:
            return None, 1.0
        mask = (torch.rand(rows, self.shape[1], device=self.get_device())
                < self.dropout_keep_probability).to(torch.uint8)
        return mask, self.dropout_keep_probability

    def compute_messages(self, sender_features, receiver_features):
        raise NotImplementedError("fused into the layer kernel: per-edge messages are never materialised")

    def combine_messages(self, forward_messages, backward_messages, self_loop_messages, previous_code,
                         mode='train'):
        raise NotImplementedError("fused into the layer kernel (normalised scatter + self loop + ReLU)")

    def compute_self_loop_messages(self, vertex_features):
        return vertex_features @ self.W_self

    def fused_layer(self, H, graph, mode):
        raise NotImplementedError

    def compute_vertex_embeddings(self, mode='train'):
        if self.vertex_embedding_function[mode] is None:
            graph = self.get_graph()
            # one-hot input (message_gcn.py:33-34, :55-56): the input is the identity, nothing below is asked for codes
            H = None if self.onehot_input else self.next_component.get_all_codes(mode=mode)[0].contiguous()
            self.vertex_embedding_function[mode] = self.fused_layer(H, graph, mode)
        return self.vertex_embedding_function[mode]

    def get_all_codes(self, mode='train'):
        collected = self.compute_vertex_embeddings(mode=mode)
        return collected, None, collected

    def get_all_subject_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)

    def get_all_object_codes(self, mode='train'):
        return self.compute_vertex_embeddings(mode=mode)
