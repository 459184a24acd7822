"""Training driver mirroring the reference's code/train.py flow (next rows N1-N3, SURVEY.md 8f):

  python -m relationprediction_b200.train --settings X.exp --dataset DIR [--max-iterations N]

settings/dataset formats, the section merge (train.py:69-86), the per-step sample transform
(graph batch -> GraphSplitSize edge dropout -> negative sampling, :201-245), loss = CE + regularisation
(:262), global-norm clipping + Adam (optimization/tensorflow_backend/algorithms.py:36-42, :65-68) and
the periodic validation MRR follow the reference; the "Converge" optimizer stack itself is replaced by
a plain loop.  Clip + Adam run on the library's kernels with the TensorFlow-1.x formulas (optim.py,
csrc/optimizer.cu)."""
import argparse
import json
import os
import queue
import threading
import time

import numpy as np

from .optim import ClippedAdam
from .common import auxilliaries, evaluation, io, model_builder, settings_reader
from .decoders.conve import ConvE
from .decoders.rotate import Rotate


def load_dataset(dataset):
    ent, rel = os.path.join(dataset, 'entities.dict'), os.path.join(dataset, 'relations.dict')
    splits = {k: io.read_triplets_as_array(os.path.join(dataset, k + '.txt'), ent, rel)
              for k in ('train', 'valid', 'test')}
    return splits, io.read_dictionary(ent), io.read_dictionary(rel)


def load_dataset_npz(path):
    """Packed form of the same data (scripts/pack_dataset.py): arrays train/valid/test [n,3] int32 in the
    dictionary ids of entities.dict / relations.dict, plus V and R.  The text datasets live in the reference
    tree, which is not present on a GPU box."""
    z = np.load(path)
    splits = {k: np.ascontiguousarray(z[k], dtype=np.int32) for k in ('train', 'valid', 'test')}
    return splits, list(range(int(z['V']))), list(range(int(z['R'])))


def sample_stream(sample, n_threads):
    """Endless stream of per-step samples; with n_threads > 0 they are produced by background threads
    (the library sampler and numpy release the GIL), so the GPU never waits for the host transform."""
    if n_threads <= 0:
        while True:
            yield sample()
    q, stop = queue.Queue(maxsize=2 * n_threads), threading.Event()

    def work():
        while not stop.is_set():
            item = sample()
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.1)
                    break
                except queue.Full:
                    pass
    threads = [threading.Thread(target=work, daemon=True) for _ in range(n_threads)]
    for t in threads:
        t.start()
    try:
        while True:
            yield q.get()
    finally:
        stop.set()


class EarlyStopper(object):
    """Stopping rule of the reference's optimizer stack (optimization/shared/algorithms.py:119-161 as configured
    by common/optimizer_parameter_parser.py:75-92): every CheckEvery iterations the validation score (filtered
    MRR) is compared with the PREVIOUS check; if it did not strictly improve and the iteration count is past
    BurninPhaseDuration, training stops; inside the burn-in the drop is ignored.  The previous score is always
    replaced by the current one (not a running best)."""

    def __init__(self, check_every, burnin=0):
        self.check_every, self.burnin = int(check_every), int(burnin)
        self.previous = None

    def due(self, iteration):
        return iteration % self.check_every == 0

    def update(self, iteration, score):
        stop = False
        if self.previous is not None and not (score > self.previous):
            if iteration > self.burnin:
                print("Stopping criterion reached.")
                stop = True
            else:
                print("Ignoring criterion while in burn-in phase.")
        self.previous = score
        return stop


def merge_settings(settings, n_entities, n_relations, n_train):
    general = settings['General']
    general.put('EntityCount', n_entities)
    general.put('RelationCount', n_relations)
    general.put('EdgeCount', n_train)
    for name in ('Encoder', 'Decoder'):
        settings[name].merge(settings['Shared'])
        settings[name].merge(general)
    settings['Optimizer'].merge(general)
    settings['Evaluation'].merge(general)
    return settings


def build_chain(settings, splits, n_entities, n_relations, device):
    """Encoder, decoder and Scorer of a run: the settings merged with the dataset sizes (train.py:69-86), the
    model built by the factory on `device` with the train split as its graph, and every split registered with the
    Scorer for the filtered metrics.  Returns (encoder, model, scorer)."""
    train = splits['train']
    merge_settings(settings, n_entities, n_relations, len(train))
    encoder = model_builder.build_encoder(settings['Encoder'], train)
    model = model_builder.build_decoder(encoder, settings['Decoder'])
    model.set_device(device)
    model.preprocess(train)
    model.register_for_test(train)
    model.initialize_train()

    scorer = evaluation.Scorer(settings['Evaluation'])
    for part in (train, splits['valid'], splits['test']):
        scorer.register_data(part)
    scorer.register_model(model)
    return encoder, model, scorer


def sample_edge_neighborhood_fast(triples, n_entities, sample_size):
    """The same sampler in the library (csrc/sampler.cu): Fenwick trees instead of an O(V) np.random.choice per
    draw (~5 s -> ~10 ms for 30 000 edges of FB15k-237); seeded from numpy's global stream."""
    import ctypes

    from . import _lib
    tri = np.ascontiguousarray(triples, dtype=np.int32)
    out = np.empty(sample_size, dtype=np.int32)
    seed = int(np.random.randint(0, 2 ** 31 - 1))
    rc = _lib.load().rgcn_sample_edge_neighborhood(ctypes.c_void_p(tri.ctypes.data), tri.shape[0], int(n_entities),
                                                   int(sample_size), seed, ctypes.c_void_p(out.ctypes.data))
    _lib.check(rc, "rgcn_sample_edge_neighborhood")
    return out


class EdgeNeighborhoodSampler(object):
    """The library sampler with the per-dataset incidence structure built once (rgcn_sampler_create); draw()
    may be called from several host threads at once.  Seeds come from numpy's global stream."""

    def __init__(self, triples, n_entities):
        import ctypes

        from . import _lib
        self._lib = _lib
        self._tri = np.ascontiguousarray(triples, dtype=np.int32)
        self._h = ctypes.c_void_p()
        rc = _lib.load().rgcn_sampler_create(ctypes.c_void_p(self._tri.ctypes.data), self._tri.shape[0],
                                             int(n_entities), ctypes.byref(self._h))
        _lib.check(rc, "rgcn_sampler_create")

    def draw(self, sample_size, seed=None):
        import ctypes
        out = np.empty(int(sample_size), dtype=np.int32)
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 31 - 1))
        rc = self._lib.load().rgcn_sampler_draw(self._h, int(sample_size), int(seed), ctypes.c_void_p(out.ctypes.data))
        self._lib.check(rc, "rgcn_sampler_draw")
        return out

    def draw_batch(self, batch, split, neg_rate, seed=None):
        """One whole training sample (graph_split [split,3], X [(neg_rate+1)*batch,3], Y) from ONE library call
        (rgcn_sampler_draw_batch): edge-neighbourhood sample, graph split and negative sampling run with the interpreter
        lock released, so sample threads do not slow the training thread down."""
        import ctypes
        batch, split, neg_rate = int(batch), int(split), int(neg_rate)
        graph_split = np.empty((split, 3), dtype=np.int32)
        X = np.empty(((neg_rate + 1) * batch, 3), dtype=np.int32)
        Y = np.empty((neg_rate + 1) * batch, dtype=np.float32)
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 31 - 1))
        rc = self._lib.load().rgcn_sampler_draw_batch(self._h, batch, split, neg_rate, int(seed),
                                                      ctypes.c_void_p(graph_split.ctypes.data),
                                                      ctypes.c_void_p(X.ctypes.data), ctypes.c_void_p(Y.ctypes.data))
        self._lib.check(rc, "rgcn_sampler_draw_batch")
        return graph_split, X, Y

    def close(self):
        if getattr(self, "_h", None):
            self._lib.load().rgcn_sampler_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown: the module globals may already be gone
            pass


def sample_edge_neighborhood(adj_list, degrees, n_triplets, sample_size):
    """Neighbourhood-expansion edge sampler (train.py:161-198), same sequential algorithm (reference
    restatement; kept as the statistical oracle of sample_edge_neighborhood_fast)."""
    edges = np.zeros(sample_size, dtype=np.int32)
    sample_counts = degrees.copy()
    picked = np.zeros(n_triplets, dtype=bool)
    seen = np.zeros(len(degrees), dtype=bool)
    for i in range(sample_size):
        weights = sample_counts * seen
        if weights.sum() == 0:
            weights = np.ones_like(weights)
            weights[sample_counts == 0] = 0
        chosen_vertex = np.random.choice(len(degrees), p=weights / weights.sum())
        chosen_adj = adj_list[chosen_vertex]
        seen[chosen_vertex] = True
        while True:
            edge_number, other = chosen_adj[np.random.randint(len(chosen_adj))]
            if not picked[edge_number]:
                break
        edges[i] = edge_number
        picked[edge_number] = True
        sample_counts[chosen_vertex] -= 1
        sample_counts[other] -= 1
        seen[other] = True
    return edges


def main(argv=None):
    ap = argparse.ArgumentParser(description="Train a model on a given dataset.")
    ap.add_argument("--settings", required=True)
    ap.add_argument("--dataset", default=None, help="directory with train/valid/test.txt + the two .dict files")
    ap.add_argument("--dataset-npz", default=None, help="the same data packed by scripts/pack_dataset.py")
    ap.add_argument("--max-iterations", type=int, default=None)
    ap.add_argument("--time-budget", type=float, default=None, help="stop training after this many seconds")
    ap.add_argument("--prefetch", type=int, default=0, help="background threads producing the per-step samples")
    ap.add_argument("--no-periodic-eval", action="store_true", help="skip the CheckEvery validation passes")
    ap.add_argument("--no-early-stopping", action="store_true",
                    help="keep the validation passes but never stop on them (only --max-iterations / --time-budget)")
    ap.add_argument("--final-eval", type=int, default=None, metavar="N",
                    help="after training rank the first N test triples (0 = all) and print one JSON line")
    ap.add_argument("--relation-metrics", action="store_true",
                    help="also rank every test triple's relation among all relations for its (head, tail) pair and "
                         "report Raw / Filtered MRR and H@1/3/10 for relation prediction after the entity metrics "
                         "(DistMult and ComplEx decoders on CUDA; refused for RotatE)")
    ap.add_argument("--set", action="append", default=[], metavar="Section.Key=Value",
                    help="override one settings entry after the file is read, e.g. "
                         "--set Encoder.NumberOfBasisFunctions=2 (repeatable)")
    ap.add_argument("--seed", type=int, default=None, help="seed numpy / torch (initial weights, samplers, dropout)")
    ap.add_argument("--dense-clip-norm", action="store_true",
                    help="clip by the norm of the summed dense gradients instead of the reference's IndexedSlices norm "
                         "(tf.clip_by_global_norm over un-aggregated per-edge slices of embedding_lookup variables)")
    ap.add_argument("--no-save", action="store_true", help="do not write checkpoints (default: the reference's "
                    "ModelSaver cadence to General.ExperimentName)")
    ap.add_argument("--save-path", default=None, help="checkpoint path prefix (default: General.ExperimentName)")
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--numpy-sampling", action="store_true",
                    help="build the graph split and the negative samples with numpy (the reference's calls) instead of "
                         "the library's one-call sample (rgcn_sampler_draw_batch)")
    ap.add_argument("--repeat-sample", action="store_true",
                    help="diagnostic: train on the FIRST sample forever (takes the host sampler out of the iteration time)")
    ap.add_argument("--profile-iterations", type=int, default=0, metavar="N",
                    help="diagnostic: after 50 warm-up iterations run N iterations with a device sync after every "
                         "phase (sample wait / forward+loss / backward / optimizer), print the mean ms per phase as one "
                         "JSON line and exit")
    args = ap.parse_args(argv)
    if (args.dataset is None) == (args.dataset_npz is None):
        ap.error("give exactly one of --dataset / --dataset-npz")

    if args.seed is not None:
        import torch
        np.random.seed(args.seed)
        torch.manual_seed(args.seed)
    settings = settings_reader.read(args.settings)
    for item in args.set:
        # dotted path into nested sections: Optimizer.Algorithm.learning_rate=0.005 reaches [Algorithm] inside
        # [Optimizer] (the settings reader nests sub-sections as Settings objects)
        path, _, value = item.partition("=")
        parts = path.split(".")
        node = settings
        for name in parts[:-1]:
            if not name or name not in node:
                ap.error("--set expects Section[.SubSection].Key=Value with existing sections, got %r" % item)
            node = node[name]
        if len(parts) < 2 or not parts[-1] or not hasattr(node, "put"):
            ap.error("--set expects Section[.SubSection].Key=Value, got %r" % item)
        node.put(parts[-1], value)
    print(settings)
    if args.dataset_npz is not None:
        splits, entities, relations = load_dataset_npz(args.dataset_npz)
    else:
        splits, entities, relations = load_dataset(args.dataset)
    train, valid, test = splits['train'], splits['valid'], splits['test']
    encoder, model, scorer = build_chain(settings, splits, len(entities), len(relations), args.device)
    general, opt = settings['General'], settings['Optimizer']
    if args.relation_metrics and isinstance(model, Rotate):
        raise SystemExit("--relation-metrics: the RotatE decoder has no relation prediction")
    if args.relation_metrics and isinstance(model, ConvE):
        raise SystemExit("--relation-metrics: the ConvE decoder has no relation prediction")

    ns = auxilliaries.NegativeSampler(int(general['NegativeSampleRate']), len(entities))
    adj_list = [[] for _ in entities]
    for i, (s, _, o) in enumerate(train.tolist()):
        adj_list[s].append((i, o))
        adj_list[o].append((i, s))
    degrees = np.array([len(a) for a in adj_list])

    edge_sampler = None
    if encoder.needs_graph() and 'GraphBatchSize' in general and int(general['GraphBatchSize']) < len(train):
        edge_sampler = EdgeNeighborhoodSampler(train, len(entities))

    # 1-N training: the step's positives are fed as X (an empty Y) and become their object and subject queries;
    # the targets come from the training split's label CSR, built here once.  No negative is drawn.
    one_to_n = model.training_objective == '1-N'
    if one_to_n:
        from . import ops
        model.set_one_to_n_labels(ops.OneToNLabels(train, len(entities), len(relations), args.device))
        print("Training objective: 1-N, label smoothing %g" % model.label_smoothing)
    if model.training_objective == 'SelfAdversarial':
        print("Training objective: SelfAdversarial, temperature %s" % model.adversarial_temperature)
    no_y = np.zeros(0, dtype=np.float32)

    def sample():
        if not encoder.needs_graph():
            if one_to_n:
                return (train, no_y)
            X, Y = ns.transform(train)
            return (X, Y)
        if edge_sampler is not None and not args.numpy_sampling:
            gbs = int(general['GraphBatchSize'])   # the whole sample in one library call (no interpreter lock held)
            split = int(float(general['GraphSplitSize']) * gbs)
            if one_to_n:   # rate 0: X is the batch itself
                graph_split, X, _ = edge_sampler.draw_batch(gbs, split, 0)
                return (graph_split, X, no_y)
            return edge_sampler.draw_batch(gbs, split, ns.negative_sample_rate)
        if 'GraphBatchSize' in general and int(general['GraphBatchSize']) < len(train):
            ids = edge_sampler.draw(int(general['GraphBatchSize']))
        else:
            ids = np.arange(len(train))
        graph_batch = train[ids]
        split = int(float(general['GraphSplitSize']) * len(graph_batch))
        graph_split = train[np.random.choice(ids, size=split, replace=False)]
        if one_to_n:
            return (graph_split, graph_batch, no_y)
        X, Y = ns.transform(graph_batch)
        return (graph_split, X, Y)

    weights = [w for w in model.get_weights()]
    algo = opt['Algorithm']
    if 'Name' in algo and str(algo['Name']).lower() != 'adam':
        # the reference also wires AdaGrad / GradientDescent (optimization/optimize.py:152-203); only the
        # Adam update is built here (both target configs use it) -- refuse instead of silently substituting it
        raise SystemExit("Optimizer.Algorithm.Name=%s is not supported by this driver (only Adam)" % algo['Name'])
    lr = float(algo['learning_rate'])
    max_norm = float(opt['MaxGradientNorm']) if 'MaxGradientNorm' in opt else None
    optimizer = ClippedAdam(weights, lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, max_norm=max_norm)
    if str(args.device).startswith("cuda"):
        from . import ops
        ops.set_slice_norms(max_norm is not None and not args.dense_clip_norm)
    report_every = int(opt['ReportTrainLossEvery']) if 'ReportTrainLossEvery' in opt else 100
    stopper = None
    if 'EarlyStopping' in opt and not args.no_periodic_eval:
        es = opt['EarlyStopping']
        stopper = EarlyStopper(es['CheckEvery'], es['BurninPhaseDuration'] if 'BurninPhaseDuration' in es else 0)
    max_it = args.max_iterations if args.max_iterations is not None else 10 ** 9
    # ModelSaver cadence of the reference (common/optimizer_parameter_parser.py:92-103): SaveEveryN, else the
    # early-stopping CheckEvery, else every iteration; path = General.ExperimentName; skipped on the stopping step
    save_every, save_path = None, None
    if not args.no_save and 'ExperimentName' in opt:
        save_path = args.save_path if args.save_path else str(opt['ExperimentName'])
        if 'SaveEveryN' in opt:
            save_every = int(opt['SaveEveryN'])
        elif 'EarlyStopping' in opt:
            save_every = int(opt['EarlyStopping']['CheckEvery'])
        else:
            save_every = 1
        if os.path.dirname(save_path):
            os.makedirs(os.path.dirname(save_path), exist_ok=True)

    # the running loss stays on the device: reading it back every iteration would serialise the host-side
    # sample transform of step i+1 behind the GPU work of step i
    running, it, last_avg = None, 0, None
    stream = sample_stream(sample, args.prefetch)
    if args.repeat_sample:
        first = next(stream)
        stream.close()
        stream = iter(lambda: first, None)
    if args.profile_iterations > 0:
        import torch
        sync = torch.cuda.synchronize if str(args.device).startswith("cuda") else (lambda: None)
        acc = {"sample_wait": 0.0, "forward_loss": 0.0, "backward": 0.0, "optimizer": 0.0}
        t_free = 0.0
        for i in range(50 + 2 * args.profile_iterations):
            timed = 50 <= i < 50 + args.profile_iterations       # phase-synchronised iterations
            free = i >= 50 + args.profile_iterations              # the same number of iterations, free-running
            if free and t_free == 0.0:
                sync()
                t_free = -time.time()
            t0 = time.time()
            batch = next(stream)
            t1 = time.time()
            optimizer.zero_grad()
            loss = model.train_loss(*batch)
            if timed:
                sync()
            t2 = time.time()
            loss.backward()
            if timed:
                sync()
            t3 = time.time()
            optimizer.step()
            if timed:
                sync()
            t4 = time.time()
            if timed:
                for k, v in zip(acc, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
                    acc[k] += v
        sync()
        t_free += time.time()
        n = args.profile_iterations
        print(json.dumps({"profile_iterations": n, "phase_ms": {k: round(v / n * 1e3, 3) for k, v in acc.items()},
                          "phase_sum_ms": round(sum(acc.values()) / n * 1e3, 3),
                          "free_running_ms_per_iteration": round(t_free / n * 1e3, 3),
                          "prefetch_threads": args.prefetch, "repeat_sample": bool(args.repeat_sample)}))
        if hasattr(stream, "close"):
            stream.close()
        return
    t_start = time.time()
    while it < max_it:
        if args.time_budget is not None and time.time() - t_start > args.time_budget:
            break
        it += 1
        optimizer.zero_grad()
        loss = model.train_loss(*next(stream))
        loss.backward()
        optimizer.step()
        running = loss.detach().clone() if running is None else running + loss.detach()
        if it == 1:
            print("Initial loss: %f" % float(running))
        if it % report_every == 0:
            last_avg = float(running) / report_every
            print("Average train loss for iteration %d-%d: %f" % (it - report_every + 1, it, last_avg))
            running = None
        if stopper is not None and stopper.due(it):
            score = scorer.compute_scores(valid).get_summary().results['Filtered']['MRR']
            print("Validation filtered MRR at iteration %d: %f" % (it, score))
            scorer.compute_scores(test).get_summary().pretty_print()
            if args.relation_metrics:
                print("Relation prediction:")
                scorer.compute_relation_mrr_scores(test).get_summary().pretty_print()
            if stopper.update(it, score) and not args.no_early_stopping:
                break
        if save_every is not None and it % save_every == 0:
            model.save(save_path)
    train_seconds = time.time() - t_start
    if hasattr(stream, "close"):
        stream.close()
    if args.final_eval is not None:
        part = test if args.final_eval == 0 else test[:args.final_eval]
        t0 = time.time()
        res = scorer.compute_scores(part).get_summary().results
        keep = ('MRR', 'H@1', 'H@3', 'H@10')
        line = {"iterations": it, "train_seconds": round(train_seconds, 2),
                "ms_per_iteration": round(train_seconds / max(it, 1) * 1e3, 3),
                "last_avg_train_loss": last_avg, "test_triples": int(len(part)),
                "eval_seconds": round(time.time() - t0, 2),
                "raw": {k: float(v) for k, v in res['Raw'].items() if k in keep},
                "filtered": {k: float(v) for k, v in res['Filtered'].items() if k in keep}}
        if args.relation_metrics:
            rel = scorer.compute_relation_mrr_scores(part).get_summary().results
            line["relation"] = {"raw": {k: float(v) for k, v in rel['Raw'].items() if k in keep},
                                "filtered": {k: float(v) for k, v in rel['Filtered'].items() if k in keep}}
        print(json.dumps(line))
    return model, scorer


if __name__ == "__main__":
    main()
