"""Generate tests/golden/interp.pt by running the REFERENCE's own record selection (interpret.py:82-212
make_feature_activation_dataset, :265-321 interpret) on the reference's own LearnedDict classes.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree):   python oracle/make_interp_golden.py

``interpret`` imports packages that are not installed here, or that would reach the network. They are replaced by
stubs at their published interfaces, carrying no selection logic:
* the imports of make_harvest_golden.py and make_metrics_golden.py (TransformerLens registry, baukit, boto3,
  matplotlib, torchtyping);
* a tiny fixed "model": ``to_tokens`` turns the sentence "g" into the 65 token ids 64 g, 64 g + 1, ... (so
  ``np.random.randint(0, n_tokens - 64)`` always starts the fragment at 0), ``run_with_cache`` returns the rows of a
  fixed activation table for those ids;
* ``datasets.load_dataset``: the sentences "0", "1", ...;
* ``neuron_explainer``: records are plain containers; ``NeuronRecord`` captures what ``interpret`` hands to the
  explainer; the explainer and simulator return canned explanations and scores.
``interpret.py`` reads ``secrets.json`` at import, so the run happens in a temporary directory holding a dummy one.
Nothing here opens a network connection.

The fixture stores the dictionaries (raw tensors with their kind, the layout of oracle/eval_oracle.py), the fragment
activations (fp16), per dictionary the reference's fp16 maxima table, its captured top records (fragment index and fp16
per-token values) per explained feature, its skipped features, and for every feature the fragments its
``sort_values(...).head(20)`` selects."""
import asyncio
import json
import os
import sys
import tempfile
import types
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_harvest_golden import HM, import_reference as import_harvest  # noqa: E402
from make_metrics_golden import import_reference as import_metrics  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "interp.pt")
L = 64


class ActivationRecord:
    def __init__(self, tokens, activations):
        self.tokens, self.activations = tokens, activations


class NeuronId:
    def __init__(self, layer_index, neuron_index):
        self.layer_index, self.neuron_index = layer_index, neuron_index


CAPTURED = []


class NeuronRecord:
    def __init__(self, neuron_id, random_sample, most_positive_activation_records):
        self.neuron_id, self.random_sample = neuron_id, random_sample
        self.most_positive_activation_records = most_positive_activation_records
        CAPTURED.append(self)

    def train_activation_records(self, slice_params):
        return self.most_positive_activation_records[:10]

    def valid_activation_records(self, slice_params):
        return self.most_positive_activation_records[10:] + self.random_sample[:5]


class Scored:
    scored_sequence_simulations = [None] * 10

    def get_preferred_score(self):
        return 0.5


class Explainer:
    def __init__(self, *a, **k):
        pass

    async def generate_explanations(self, **k):
        return ["canned explanation"]


def stub_neuron_explainer():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m

    async def simulate_and_score(simulator, records):
        return Scored()

    for pkg in ("neuron_explainer", "neuron_explainer.activations", "neuron_explainer.explanations"):
        mod(pkg)
    mod("neuron_explainer.activations.activation_records",
        calculate_max_activation=lambda recs: max(max(r.activations) for r in recs))
    mod("neuron_explainer.activations.activations", ActivationRecord=ActivationRecord, NeuronId=NeuronId,
        NeuronRecord=NeuronRecord, ActivationRecordSliceParams=lambda **k: SimpleNamespace(**k))
    mod("neuron_explainer.explanations.calibrated_simulator", UncalibratedNeuronSimulator=lambda sim: sim)
    mod("neuron_explainer.explanations.explainer", TokenActivationPairExplainer=Explainer)
    mod("neuron_explainer.explanations.prompt_builder",
        PromptFormat=SimpleNamespace(HARMONY_V4="harmony_v4", INSTRUCTION_FOLLOWING="instruction_following"))
    mod("neuron_explainer.explanations.scoring", simulate_and_score=simulate_and_score,
        aggregate_scored_sequence_simulations=lambda sims: Scored())
    mod("neuron_explainer.explanations.simulator", ExplanationNeuronSimulator=lambda *a, **k: None)
    mod("neuron_explainer.fast_dataclasses", loads=json.loads)


class TinyModel:
    """Token id 64 g + t stands for row t of fragment g; the cache returns that row of the activation table."""

    def __init__(self, table):
        self.cfg = SimpleNamespace(model_name=HM.TINY_TL_NAME)
        self.table = table

    def to(self, device):
        return self

    def eval(self):
        return self

    def to_tokens(self, text, prepend_bos=False):
        return (torch.arange(L + 1) + int(text) * L)[None]

    def to_str_tokens(self, tokens):
        return [f"t{int(t)}" for t in tokens]

    def run_with_cache(self, tokens):
        return None, _Cache(self.table[tokens])


class _Cache:
    def __init__(self, acts):
        self.acts = acts

    def __getitem__(self, name):
        return self.acts


def main():
    import_harvest()
    _, ld, topk = import_metrics()
    stub_neuron_explainer()
    g = torch.Generator().manual_seed(int(os.environ.get("INTERP_GOLDEN_SEED", 10)))
    rn = lambda *s: torch.randn(*s, generator=g)
    d, n_frag = 16, 64
    # fragments with their own scale, spread over two decades: a feature's activity varies from fragment to fragment,
    # and neighbouring fragment maxima differ by far more than fp16's resolution. Stored as fp16, the reference's
    # activation chunk format; the model serves them as fp32.
    x = rn(n_frag, L, d) * torch.exp(torch.rand(n_frag, 1, 1, generator=g) * 5.0 - 3.0)
    acts = x.reshape(n_frag * L, d).half()
    bias = -torch.linspace(1.0, 25.0, 37)        # later features fire only in the largest fragments
    bias[3] = -1e3                                             # a feature that never fires
    dicts = {"tied_odd": {"kind": "tied", "encoder": rn(37, d), "encoder_bias": bias},   # n not a multiple of 8
             "untied": {"kind": "untied", "encoder": rn(24, d) * 0.3, "encoder_bias": -torch.linspace(0.5, 3.0, 24),
                        "decoder": rn(24, d)},
             "topk": {"kind": "topk", "dict": topk.TopKEncoder.to_learned_dict({"dict": rn(32, d)},
                                                                               {"sparsity": torch.tensor(4)}).dict,
                      "sparsity": 4}}

    def make(e):
        if e["kind"] == "tied":
            return ld.TiedSAE(e["encoder"], e["encoder_bias"], norm_encoder=True)
        if e["kind"] == "untied":
            return ld.UntiedSAE(e["encoder"], e["decoder"], e["encoder_bias"])
        return topk.TopKLearnedDict(e["dict"], e["sparsity"])

    out = {"dicts": dicts, "acts": acts, "fragment_len": L, "n_examples": 20, "cases": {}}
    with tempfile.TemporaryDirectory() as tmp:
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            with open("secrets.json", "w") as f:
                json.dump({"openai_key": "unused"}, f)
            import interpret as I
            assert I.OPENAI_FRAGMENT_LEN == L and I.TOTAL_EXAMPLES == 20
            I.load_dataset = lambda *a, **k: [{"text": str(i)} for i in range(n_frag + 40)]
            # the reference encodes whole batches of 20 sentences and keeps the first n_frag: the sentences past them
            # get zero rows
            table = torch.cat([acts.float(), torch.zeros(40 * L + 1, d)])
            for name, e in dicts.items():
                CAPTURED.clear()
                torch.manual_seed(0)
                np.random.seed(0)
                n = e["encoder"].shape[0] if "encoder" in e else e["dict"].shape[0]
                with torch.no_grad():
                    df = I.make_feature_activation_dataset(TinyModel(table), make(e), layer=2, layer_loc="residual",
                                                           device="cpu", n_fragments=n_frag)
                ids = [int(t[0][1:]) // L for t in df["fragment_token_strs"]]
                assert ids == list(range(n_frag))
                asyncio.run(I.interpret(df, os.path.join(tmp, name), n_feats_to_explain=n))
                maxes = torch.tensor(np.stack([df[f"feature_{f}_max"].to_numpy() for f in range(n)], 1))
                top = {}
                for rec in CAPTURED:
                    recs = rec.most_positive_activation_records
                    top[rec.neuron_id.neuron_index] = {
                        "fragments": torch.tensor([int(r.tokens[0][1:]) // L for r in recs]),
                        "activations": torch.tensor(np.array([np.array(r.activations, dtype=np.float16) for r in recs]))}
                head = torch.stack([torch.tensor(df.sort_values(by=f"feature_{f}_max", ascending=False)
                                                 .head(I.TOTAL_EXAMPLES).index.to_numpy()) for f in range(n)])
                skipped = torch.tensor([f not in top for f in range(n)])
                # positive fp16 maxima have no ties at the top-20 boundary (the reference's order there is unspecified)
                srt = maxes.float().sort(0, descending=True).values
                tie = (srt[19] == srt[20]) & (srt[19] > 0)
                assert not bool(tie.any()), (name, tie.nonzero().flatten().tolist())
                out["cases"][name] = {"maxes": maxes, "top": top, "head": head, "skipped": skipped}
                n_act = (maxes > 0).sum(0)
                print(name, "explained", len(top), "skipped", int(skipped.sum()), "active fragments min/max",
                      int(n_act.min()), int(n_act.max()))
        finally:
            os.chdir(cwd)
    torch.save(out, OUT)
    print("wrote", os.path.normpath(OUT), os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
