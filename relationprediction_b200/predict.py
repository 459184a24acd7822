"""Top-k entity and relation prediction from a trained checkpoint:

  python -m relationprediction_b200.predict --settings X.exp --dataset DIR | --dataset-npz F --checkpoint PATH
                                            --queries FILE --k K [--raw] --out FILE

builds the model as the training driver does (train.build_chain), loads the weights Model.save wrote, and answers
every query of FILE, one per line:

  head<TAB>relation<TAB>?      the K most likely tails
  ?<TAB>relation<TAB>tail      the K most likely heads
  head<TAB>?<TAB>tail          the K most likely relations linking head to tail

Names come from the dataset's entities.dict / relations.dict; with --dataset-npz they are numeric ids.  By default
the answers leave out every entity (or relation) that completes a triple of the train, valid or test split (the
filtered setting of the evaluation); --raw keeps them.  The output has one line per answer:

  query_index<TAB>position<TAB>answer<TAB>score

query_index counts the queries from 0 in file order, position counts from 1, and score is the model's sigmoid
score.  The answer is an entity name, or a relation name for a relation query.  A query with fewer than K eligible
answers gets fewer lines."""
import argparse

import numpy as np

from . import train as driver
from .common import settings_reader


class QueryError(ValueError):
    pass


def parse_queries(lines, entity_ids, relation_ids):
    """[(s, r, o, side)] with the unknown field as -1 and side 0 = predict the head, 1 = predict the tail,
    2 = predict the relation.  entity_ids / relation_ids map names to ids.  Blank lines are skipped; anything else
    malformed raises QueryError naming the line."""
    out = []
    for no, line in enumerate(lines, 1):
        line = line.rstrip("\r\n")
        if not line.strip():
            continue
        f = [x.strip() for x in line.split("\t")]
        if len(f) != 3:
            raise QueryError("line %d: expected head<TAB>relation<TAB>?, ?<TAB>relation<TAB>tail or "
                             "head<TAB>?<TAB>tail, got %r" % (no, line))
        if f.count("?") != 1:
            raise QueryError("line %d: exactly one of head, relation and tail must be '?', got %r" % (no, line))
        if f[1] == "?":
            for name in (f[0], f[2]):
                if name not in entity_ids:
                    raise QueryError("line %d: unknown entity %r" % (no, name))
            out.append((entity_ids[f[0]], -1, entity_ids[f[2]], 2))
            continue
        if f[1] not in relation_ids:
            raise QueryError("line %d: unknown relation %r" % (no, f[1]))
        side = 0 if f[0] == "?" else 1
        known = f[2] if side == 0 else f[0]
        if known not in entity_ids:
            raise QueryError("line %d: unknown entity %r" % (no, known))
        e = entity_ids[known]
        out.append((-1, relation_ids[f[1]], e, 0) if side == 0 else (e, relation_ids[f[1]], -1, 1))
    return out


def answer(scorer, queries, k, filtered):
    """[(query_index, position, answer id, score)] for the parsed queries: entity queries through
    Scorer.predict_top_k, one call per side, and relation queries (side 2, answer = a relation id) through
    Scorer.predict_top_k_relations, one call.  The unknown field is given an id in range (the fused paths do not
    read it): the known entity's for an entity query, 0 for a relation query."""
    rows = []
    for side in (0, 1, 2):
        idx = [i for i, q in enumerate(queries) if q[3] == side]
        if not idx:
            continue
        tri = np.array([queries[i][:3] for i in idx], dtype=np.int64)
        if side == 2:
            tri[:, 1] = 0
            ids, _, scores = scorer.predict_top_k_relations(tri, k, filtered=filtered)
        else:
            unknown = 0 if side == 0 else 2
            tri[:, unknown] = tri[:, 2 - unknown]
            ids, _, scores = scorer.predict_top_k(tri, k, side, filtered=filtered)
        for j, qi in enumerate(idx):
            for p in range(ids.shape[1]):
                if ids[j, p] < 0:
                    break
                rows.append((qi, p + 1, int(ids[j, p]), float(scores[j, p])))
    rows.sort(key=lambda r: (r[0], r[1]))
    return rows


def main(argv=None):
    ap = argparse.ArgumentParser(description="Predict the K most likely entities for (head, relation, ?) and "
                                             "(?, relation, tail) queries, and the K most likely relations for "
                                             "(head, ?, tail) queries, with a trained model.")
    ap.add_argument("--settings", required=True)
    ap.add_argument("--dataset", default=None, help="directory with train/valid/test.txt + the two .dict files")
    ap.add_argument("--dataset-npz", default=None, help="the same data packed by scripts/pack_dataset.py "
                                                        "(queries then name entities and relations by id)")
    ap.add_argument("--checkpoint", required=True, help="a file written by Model.save (PREFIX-N.pt)")
    ap.add_argument("--queries", required=True, help="one query per line: head<TAB>relation<TAB>?, "
                                                     "?<TAB>relation<TAB>tail or head<TAB>?<TAB>tail")
    ap.add_argument("--k", type=int, required=True, help="answers per query, 1 <= K <= 128")
    ap.add_argument("--raw", action="store_true", help="keep entities (relations) that complete a known triple")
    ap.add_argument("--out", required=True, help="output file: query_index<TAB>position<TAB>answer<TAB>score, the "
                                                "answer an entity, or a relation for head<TAB>?<TAB>tail")
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)
    if (args.dataset is None) == (args.dataset_npz is None):
        ap.error("give exactly one of --dataset / --dataset-npz")
    if not 1 <= args.k <= 128:
        ap.error("--k must be in [1, 128], got %d" % args.k)

    settings = settings_reader.read(args.settings)
    if args.dataset_npz is not None:
        splits, entities, relations = driver.load_dataset_npz(args.dataset_npz)
        ent_names = {str(i): i for i in entities}
        rel_names = {str(i): i for i in relations}
        name_of = rel_name_of = str
    else:
        splits, entities, relations = driver.load_dataset(args.dataset)
        ent_names = {v: i for i, v in entities.items()}
        rel_names = {v: i for i, v in relations.items()}
        name_of, rel_name_of = entities.__getitem__, relations.__getitem__
    with open(args.queries) as fh:
        try:
            queries = parse_queries(fh, ent_names, rel_names)
        except QueryError as e:
            ap.error("%s: %s" % (args.queries, e))

    _, model, scorer = driver.build_chain(settings, splits, len(entities), len(relations), args.device)
    model.load(args.checkpoint)
    rows = answer(scorer, queries, args.k, filtered=not args.raw)
    with open(args.out, "w") as fh:
        for qi, pos, ans, score in rows:
            name = rel_name_of(ans) if queries[qi][3] == 2 else name_of(ans)
            fh.write("%d\t%d\t%s\t%.9g\n" % (qi, pos, name, score))
    return rows


if __name__ == "__main__":
    main()
