"""Float64 restatement of the variational head (extras/variational_encoding.py:14-31) -- TEST INFRASTRUCTURE.

  mu, l = (W_mu, W_sigma)                          H is None (variational_embedding)
          (H W_mu + b_mu, H W_sigma + b_sigma)     otherwise (variational_gcn_basis)
  z  = mu + exp(l) eps,   kl = -0.0005 sum(1 + 2 l - mu^2 - exp(2 l))

`variational` is differentiable through torch autograd; `gradients` states the closed-form gradients the CUDA
backward implements, so a test can check one against the other."""
import torch


def mu_log_sigma(H, W_mu, b_mu, W_sigma, b_sigma):
    if H is None:
        return W_mu, W_sigma
    return H @ W_mu + b_mu, H @ W_sigma + b_sigma


def variational(H, W_mu, b_mu, W_sigma, b_sigma, eps):
    mu, ls = mu_log_sigma(H, W_mu, b_mu, W_sigma, b_sigma)
    z = mu + torch.exp(ls) * eps.to(mu.dtype)
    kl = -0.0005 * torch.sum(1 + 2 * ls - mu ** 2 - torch.exp(2 * ls))
    return z, kl


def gradients(H, W_mu, b_mu, W_sigma, b_sigma, eps, dz, g):
    """(dH, dW_mu, db_mu, dW_sigma, db_sigma) for incoming dz and KL gradient g; dH and the db are None for H None."""
    mu, ls = mu_log_sigma(H, W_mu, b_mu, W_sigma, b_sigma)
    dmu = dz + 0.001 * g * mu
    dls = dz * torch.exp(ls) * eps.to(mu.dtype) + 0.001 * g * (torch.exp(2 * ls) - 1)
    if H is None:
        return None, dmu, None, dls, None
    return dmu @ W_mu.T + dls @ W_sigma.T, H.T @ dmu, dmu.sum(0), H.T @ dls, dls.sum(0)


def weight_names(model):
    """Names of model.get_weights() in the golden generator's spelling: the class path from the top of the chain
    (a split's branches as /mu and /sigma, a shared trunk named along /mu), '#', the index in local_get_weights()."""
    names = {}

    def walk(comp, path):
        while comp is not None:
            path = path + "/" + comp.__class__.__name__
            for i, w in enumerate(comp.local_get_weights() if hasattr(comp, 'local_get_weights') else []):
                names.setdefault(id(w), "%s#%d" % (path, i))
            if hasattr(comp, 'next_components'):
                walk(comp.mu_network, path + "/mu")
                walk(comp.sigma_network, path + "/sigma")
                return
            comp = comp.next_component
    walk(model, "")
    return [names[id(w)] for w in model.get_weights()]
