"""Writes tests/golden/reference_main_toyset.json: the result file and the metrics file that the reference's own
``main`` (biencoder/beir/beir_dense_retriever.py, run unmodified on the stand-in ``beir`` / ``custommodels`` packages of
sgpt_b200/compat with the CPU stand-ins of tests/test_reference_main_cpu.py) writes for the toy BEIR set of that test.

  python tests/golden/make_reference_main.py <path of the reference's beir_dense_retriever.py>
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def main(ref_script):
    from sgpt_b200.compat.run_reference import load_reference_script
    from tests.test_reference_main_cpu import _CpuDRES, _ToyEmbedder, make_toy_beir

    with tempfile.TemporaryDirectory() as tmp:
        make_toy_beir(tmp)
        os.chdir(tmp)  # main writes its result files into the working directory
        mod = load_reference_script(ref_script, embedder_cls=_ToyEmbedder, module_name="ref_bdr_golden")
        mod.DenseRetrievalExactSearch = _CpuDRES  # (bound at import: `from custommodels import ...`)
        sys.argv = ["beir_dense_retriever.py", "--dataset", "toyset", "--datapath", os.path.join(tmp, "datasets"),
                    "--modelname", "toy/model", "--method", "weightedmean", "--device", "cpu", "--batchsize", "16", "--specb"]
        mod.main(mod.parse_args())
        results = json.load(open(os.path.join(tmp, "results_toy_model_weightedmean_toyset.json")))
        metrics = json.load(open(os.path.join(tmp, "beir_embeddings_ndcgs.json")))
    out = os.path.join(HERE, "reference_main_toyset.json")
    with open(out, "w") as f:
        json.dump({"results": results, "metrics": metrics}, f, sort_keys=True)
    print("wrote", out)


if __name__ == "__main__":
    main(sys.argv[1])
