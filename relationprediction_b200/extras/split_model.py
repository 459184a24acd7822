"""SplitModel: a component with several branches that may share the components below them (reference:
split_model.py:7-70, the base of VariationalEncoding).

The reference collects the branches' weights and input variables with list(set(...)), so their order is whatever the
set gives, and it runs initialize_train down every branch, which initialises a shared trunk once per branch.  Here
every component below the split is reached exactly once, in a fixed order: branch by branch, each branch contributing
the components no earlier branch reached.  For the collecting calls (get_weights, the input lists, get_regularization)
that is the first branch's whole chain deepest first (the shared trunk, then the first branch's own components), then
each further branch's own components, deepest first, then this component's own.  `next_component` is the first
branch, so the forwarding calls (get_graph, get_device) go down it."""
import torch

from ..model import Model


class SplitModel(Model):
    def __init__(self, next_component_list, settings):
        self.next_components = list(next_component_list)
        Model.__init__(self, self.next_components[0], settings)

    def needs_graph(self):
        return any(c.needs_graph() for c in self.next_components)

    def branch_parts(self):
        """Per branch, the components it reaches that no earlier branch reached, top-down."""
        seen, parts = set(), []
        for comp in self.next_components:
            own = []
            while comp is not None and id(comp) not in seen:
                seen.add(id(comp))
                own.append(comp)
                comp = comp.next_component
            parts.append(own)
        return parts

    def set_device(self, device):
        self.device = torch.device(device)
        for own in self.branch_parts():
            for comp in own:
                comp.device = self.device

    def __local_run_delegate__(self, name, *args, **kw):
        hook = getattr(self, 'local_' + name, None)
        if hook is not None:
            hook(*args, **kw)
        for own in self.branch_parts():
            for comp in own:
                hook = getattr(comp, 'local_' + name, None)
                if hook is not None:
                    hook(*args, **kw)

    def __local_expand_delegate__(self, name, *args, base=None, **kw):
        result = [] if base is None else base
        for own in self.branch_parts():
            for comp in reversed(own):
                hook = getattr(comp, 'local_' + name, None)
                if hook is not None:
                    result = result + hook(*args, **kw)
        hook = getattr(self, 'local_' + name, None)
        return result + hook(*args, **kw) if hook is not None else result
