"""Generate ``tests/golden/eraser_latex.npz``: the LaTeX files of the UNMODIFIED reference pipeline on CPU (authoring
container).

    python -m oracle.make_golden_eraser_latex    # from the repo root, needs /root/reference and transformers

TEST INFRASTRUCTURE.  The pipeline's test loop (``bert_pipeline.py:469-561``) lives inside ``main()``, after training, so
this script takes the loop body's statements out of the reference's own source (``ast``) and executes them, unchanged,
per annotation and mode, with the names they read bound here: ``method_expl`` calls the reference ``Generator`` methods
through ``ref_harness`` (batch 1), ``preds`` holds the ``layers_ours`` classifier's logits, ``args.output_dir`` is
``out``, relative to a temporary working directory (``generate_all`` writes into the working directory itself; its files
are recorded under ``generate_all/``).  The data are those of
``make_golden_eraser.py``: its seeded vocabulary, documents and annotations, a real ``BertTokenizer`` and the tiny BERT of
``bert_tiny.npz`` (``generate_LRP`` with start_layer 2).  Recorded: the target and counterfactual maps the reference
passed to ``generate()``, the logits, the bytes of every file, and ``generate()`` applied to hand-built rows (constant
rows, ties, values around the 1 % cut, a single token, LaTeX-special tokens and ``##`` pieces, NaN, infinities, negative
values).  The annotations' evidence groups iterate in hash order, so the script re-runs itself with PYTHONHASHSEED=0.
"""
import ast
import json
import os
import subprocess
import sys
import tempfile
import types
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh              # noqa: E402
from oracle import make_golden_eraser as mge      # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "eraser_latex.npz")
OUTPUT_DIR = "out"                                # the --output_dir the figure page's paths are built from
CLASSES = mge.CLASSES


def loop_statements(rpipe):
    """The statements of the reference's per-annotation loop body (``for s in batch_elements``), split by mode."""
    with open(rpipe.__file__) as f, warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)                  # the reference's "\i" / "\#" string escapes
        tree = ast.parse(f.read())
    main = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "main")
    loop = next(n for n in ast.walk(main) if isinstance(n, ast.For) and isinstance(n.target, ast.Name)
                and n.target.id == "s")
    folder = next(n for n in ast.walk(main) if isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Name)
                  and n.targets[0].id == "method_folder")

    def mode_if(name):
        return next(n for n in loop.body if isinstance(n, ast.If) and isinstance(n.test, ast.Compare)
                    and getattr(n.test.comparators[0], "value", None) == name)
    body = loop.body
    head = body[:4]                                                  # doc_name, inp, classification, correct
    gen_all, gt = mode_if("generate_all"), mode_if("ground_truth")
    start = body.index(gt) + 1                                       # text = convert_ids_to_tokens(...) ...
    end = next(i for i, n in enumerate(body) if isinstance(n, ast.If) and i > start) + 1   # ... through the CF block

    def code(stmts):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SyntaxWarning)
            return compile(ast.fix_missing_locations(ast.Module(body=list(stmts), type_ignores=[])), rpipe.__file__,
                           "exec")
    strip = lambda stmts: [n for n in stmts if not isinstance(n, (ast.Break, ast.AugAssign)) and not (  # noqa: E731
        isinstance(n, ast.Assign) and isinstance(n.targets[0], ast.Name) and n.targets[0].id == "j")]
    return {"folder": code([folder]), "head": code(head), "generate_all": code(strip(gen_all.body)),
            "ground_truth": code(strip(gt.body)), "method": code(body[start:end])}


def hand_rows():
    """(tokens, values) rows the models do not produce; generate() sees them unclamped."""
    f = np.float32
    cut = [float(np.nextafter(f(0.01), f(0)) if k < 0 else f(0.01)) for k in (-1, 0)]
    ulps = [float(x) for x in (f(0.01) + np.arange(-3, 4, dtype=np.float32) * np.spacing(f(0.01)))]
    special = ["[CLS]", "$100", "50%", "a&b", "x^2", "#1", "snake_case", "{x}", "back\\slash", "play", "##ing", "##",
               "$", "a$b$c", "[SEP]"]
    g = np.random.default_rng(7)
    rows = [(["a", "b", "c", "d"], [0.5] * 4),                                      # constant
            (["a", "b", "c"], [0.0, 0.0, 0.0]),
            (["x"], [0.7]),                                                         # a single token
            (["a", "b", "c", "d", "e"], [0.2, 0.9, 0.2, 0.9, 0.5]),                 # ties at min and max
            (["t%d" % i for i in range(11)], [0.0, 1.0] + cut + ulps),              # around the 1 % cut
            (["t%d" % i for i in range(6)], [0.0, 100.0, 1.0, 0.999999, 1.000001, 0.99]),
            (special, [float(x) for x in g.random(len(special), dtype=np.float32)]),
            (["a", "b", "c", "d"], [0.1, float("nan"), 0.5, -0.2]),                 # NaN
            (["a", "b"], [float("nan"), float("nan")]),
            (["a", "b", "c"], [1.0, float("inf"), 2.0]),                            # infinities
            (["a", "b", "c"], [float("-inf"), 0.5, 2.0]),
            (["a", "b", "c"], [-3e38, 3e38, 0.0]),                                  # max - min overflows
            (["a", "b", "c", "d", "e"], [-0.5, -0.25, -0.0, 0.0, -1.0]),            # negative values, signed zeros
            (["l%d" % i for i in range(300)], [float(x) for x in g.standard_normal(300, dtype=np.float32)])]
    return rows


def run():
    from transformers import BertTokenizer
    vocab = mge.vocabulary()
    docs = mge.documents(vocab)
    ann_lines = mge.annotations(docs)
    out = {"vocab": np.array(vocab), "docids": np.array(sorted(docs)), "docs": np.array([docs[d] for d in sorted(docs)]),
           "annotations": np.array(ann_lines), "max_length": np.int64(mge.MAX_LENGTH), "output_dir": np.array(OUTPUT_DIR),
           "hashseed": np.array(os.environ["PYTHONHASHSEED"])}
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, "vocab.txt"), "w") as f:
            f.write("".join(v + "\n" for v in vocab))
        tok = BertTokenizer(os.path.join(tmp, "vocab.txt"), do_lower_case=True)
        data = os.path.join(tmp, "data")
        os.makedirs(os.path.join(data, "docs"))
        for d, text in docs.items():
            with open(os.path.join(data, "docs", d), "w") as f:
                f.write(text)
        with open(os.path.join(data, "test.jsonl"), "w") as f:
            f.write("".join(line + "\n" for line in ann_lines))
        rh._prepare_bert_imports()
        with rh._ref_imports():
            from BERT_rationale_benchmark import utils as rutils
            from BERT_rationale_benchmark.models.pipeline import bert_pipeline as rpipe
            stmts = loop_statements(rpipe)
            test = rutils.annotations_from_jsonl(os.path.join(data, "test.jsonl"))
            texts = rutils.load_documents(data, set(docs))
            enc = {d: tok(texts[d], add_special_tokens=True, max_length=mge.MAX_LENGTH, return_token_type_ids=False,
                          padding=False, return_attention_mask=True, return_tensors="pt", truncation=True) for d in texts}
            p = mge.params()
            models = {kind: mge.build(kind, p) for kind in ("ours", "cls_lrp")}
            classes = {c: i for i, c in enumerate(CLASSES)}
            cwd = os.path.join(tmp, "cwd")                         # out/<folder>/... and generate_all's files
            os.makedirs(cwd)
            ns = {"os": os, "torch": torch, "args": types.SimpleNamespace(output_dir=OUTPUT_DIR), "tokenizer": tok,
                  "documents": texts, "generate": rpipe.generate, "get_input_words": rpipe.get_input_words,
                  "extract_docid_from_dataset_element": rpipe.extract_docid_from_dataset_element,
                  "extract_evidence_from_dataset_element": rpipe.extract_evidence_from_dataset_element}
            exec(stmts["folder"], ns)
            old = os.getcwd()
            os.chdir(cwd)
            for m in ns["method_folder"].values():
                os.makedirs(os.path.join(OUTPUT_DIR, m), exist_ok=True)
            try:
                for j, s in enumerate(test):
                    d = rpipe.extract_docid_from_dataset_element(s)
                    ids, mask = enc[d]["input_ids"], enc[d]["attention_mask"]
                    out["ids.%d" % j] = ids[0].numpy().astype(np.int64)
                    out["pieces.%d" % j] = np.array(tok.convert_ids_to_tokens(ids[0]))
                    logits = rh.bert_logits(models["ours"], ids, mask)
                    out["logits.%d" % j] = logits[0].numpy()
                    ns.update(s=s, j=j, input_ids=ids, attention_masks=mask, preds=logits,
                              targets=torch.tensor([classes[s.classification]]))
                    for mode in ("generate_all", "ground_truth") + tuple(m for m, *_ in mge.METHODS):
                        ns["method"] = mode
                        exec(stmts["head"], ns)
                        if mode in ("generate_all", "ground_truth"):
                            exec(stmts[mode], ns)
                            continue
                        _, kind, which, kw = next(x for x in mge.METHODS if x[0] == mode)
                        maps = {}

                        def expl(input_ids, attention_mask, index, _m=models[kind], _w=which, _kw=kw, _maps=maps):
                            r = rh.bert_generate(_m, input_ids, attention_mask, _w, index=index, **_kw)
                            _maps[index] = r[0].numpy().copy()
                            return r
                        ns["method_expl"] = {mode: expl}
                        exec(stmts["method"], ns)
                        t = classes[s.classification]
                        out["%s.map.%d" % (mode, j)] = maps[t]
                        if 1 - t in maps:
                            out["%s.cf_map.%d" % (mode, j)] = maps[1 - t]
            finally:
                os.chdir(old)
            files = []
            for dirpath, _, names in os.walk(cwd):
                for name in names:
                    rel = os.path.relpath(os.path.join(dirpath, name), cwd)
                    rel = rel[len(OUTPUT_DIR) + 1:] if rel.startswith(OUTPUT_DIR + os.sep) else "generate_all/" + rel
                    with open(os.path.join(dirpath, name), "rb") as f:
                        out["file." + rel] = np.frombuffer(f.read(), dtype=np.uint8)
                    files.append(rel)
            out["files"] = np.array(sorted(files))
            for i, (tokens, values) in enumerate(hand_rows()):
                path = os.path.join(tmp, "hand_%d.tex" % i)
                rpipe.generate(tokens, torch.tensor(values, dtype=torch.float32), path)
                out["hand.tokens.%d" % i] = np.array(tokens)
                out["hand.values.%d" % i] = np.array(values, dtype=np.float32)
                with open(path, "rb") as f:
                    out["hand.file.%d" % i] = np.frombuffer(f.read(), dtype=np.uint8)
            out["hand.count"] = np.int64(len(hand_rows()))
    np.savez_compressed(OUT, **out)
    print("eraser_latex.npz", len(out), "arrays,", len(files), "files,", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    if os.environ.get("PYTHONHASHSEED") != "0":
        sys.exit(subprocess.call([sys.executable, "-m", "oracle.make_golden_eraser_latex"], cwd=ROOT,
                                 env=dict(os.environ, PYTHONHASHSEED="0")))
    torch.set_num_threads(os.cpu_count())
    run()
