"""The final-hidden-state criterion of tests/layer_parity.py, checked without a GPU at tiny Llama / Qwen2 / Qwen3 shapes
(6 rows of 1..~200 tokens, 6 forced steps): the identity LM head reads the hidden state exactly, the seeded weights give
layer updates of the residual stream's size, the permuted twin passes (it is a legitimate bf16 implementation) and every
negative control fails (the criterion sees a 2^-4 error in one head, one norm block or one RoPE position).

Measured here (transformers 5.5, CPU), worst ratios (row / block / element; A = 2, M = 4 make the limits 2 / 2 / 1):

  shape       twin                  controls: row ratio (does the old logits check catch it?)
  tiny_g2     1.13 / 1.17 / 0.33    v head 6.0 (yes), o head 3.4 (yes), final norm 3.8 (block 7.4; yes), rope 25.8 (yes)
  tiny_qwen2  1.10 / 1.20 / 0.38    v head 4.9 (yes), o head 2.9 (no), final norm 3.6 (block 6.6; yes), rope 25.5 (yes),
                                    q bias 22.8 (yes)
  tiny_qwen3  1.28 / 1.30 / 0.33    v head 4.6 (yes), o head 2.4 (yes), final norm 3.7 (block 7.5; yes), rope 22.1 (yes),
                                    k_norm 4.2 (yes)

At these tiny widths the old check (4 ulps of the largest logit through a random head) catches most controls too; what
it cannot do is tell which rows, steps or columns are off, and it is blind below its 4-ulp floor."""
import collections

import pytest
import torch

import layer_parity as LP

T = 6
SHAPES = ["tiny_g2", "tiny_qwen2", "tiny_qwen3"]
SEED = 1


@pytest.fixture(scope="module")
def cases():
    """per shape: weights, rows, and the float64 / bf16 / twin final hidden states, computed once"""
    torch.set_num_threads(max(1, min(8, torch.get_num_threads())))
    out = {}

    def get(shape):
        if shape not in out:
            cfg = LP.config(shape)
            H = cfg["hidden_size"]
            sd = LP.draw_weights(cfg, SEED)
            prompts = LP.prompt_pool(6, H, 5, fixed=(1, 64, 65, 129), hi=200)
            seqs = LP.sequences(prompts, LP.forced_tokens(len(prompts), T, H, 5), T)
            m64 = LP.build_hf(cfg, sd, torch.float64)
            updates = _update_ratios(m64, seqs)
            ref = torch.stack(LP.run_rows(m64, seqs, T))
            del m64
            hf = torch.stack(LP.run_rows(LP.build_hf(cfg, sd, torch.bfloat16), seqs, T))
            p, q = LP.permutations(cfg, SEED)
            twin = torch.stack(LP.run_rows(LP.build_hf(cfg, LP.permute(sd, p, q), torch.bfloat16), seqs, T))[..., torch.argsort(p)]
            out[shape] = dict(cfg=cfg, sd=sd, seqs=seqs, ref=ref, hf=hf, twin=twin, updates=updates)
        return out[shape]
    return get


def _update_ratios(model, seqs):
    """rms(attention / MLP output) over rms(the residual stream entering that block), per layer, block and row"""
    got = collections.defaultdict(list)
    hooks = []
    for i, layer in enumerate(model.model.layers):
        state = {}
        hooks.append(layer.register_forward_pre_hook(
            lambda mod, args, kw, st=state: st.update(x=kw.get("hidden_states", args[0] if args else None)), with_kwargs=True))

        def attn(mod, args, out, st=state, i=i):
            o = out[0] if isinstance(out, tuple) else out
            got[(i, "attn")].append(float(o.pow(2).mean().sqrt() / st["x"].pow(2).mean().sqrt()))
            st["mid"] = st["x"] + o

        def mlp(mod, args, out, st=state, i=i):
            got[(i, "mlp")].append(float(out.pow(2).mean().sqrt() / st["mid"].pow(2).mean().sqrt()))
        hooks += [layer.self_attn.register_forward_hook(attn), layer.mlp.register_forward_hook(mlp)]
    try:
        LP.run_rows(model, seqs, T)
    finally:
        for h in hooks:
            h.remove()
    return got


@pytest.mark.parametrize("shape", SHAPES)
def test_identity_head_logits_are_the_final_hidden_state(cases, shape):
    """bf16 transformers model with lm_head = eye(H): its logits equal its final-normed hidden state bit for bit"""
    c = cases(shape)
    model = LP.build_hf(c["cfg"], c["sd"], torch.bfloat16)
    ids = torch.tensor(c["seqs"][3])[None]
    with torch.no_grad():
        out = model(input_ids=ids, output_hidden_states=True)
    h = model.model(input_ids=ids).last_hidden_state
    assert out.logits.shape[-1] == c["cfg"]["hidden_size"]
    assert torch.equal(out.logits.to(torch.bfloat16).view(torch.int16), h.view(torch.int16))


@pytest.mark.parametrize("shape", SHAPES)
def test_layer_updates_comparable_to_the_residual_stream(cases, shape):
    c = cases(shape)
    lo, hi = LP.UPDATE_RMS_RANGE
    for key, r in c["updates"].items():
        assert lo <= min(r) and max(r) <= hi, f"{key}: update / residual rms in [{min(r):.2f}, {max(r):.2f}]"


@pytest.mark.parametrize("shape", SHAPES)
def test_permuted_twin_passes(cases, shape):
    c = cases(shape)
    r = LP.judge(c["twin"], c["hf"], c["ref"])
    print(f"{shape} twin: {LP.fmt(r)}")
    assert r["ok"], LP.fmt(r)
    assert not torch.equal(c["twin"], c["hf"]), "the twin must sum in another order than the yardstick"


CONTROLS = [(s, n) for s in SHAPES for n in LP.controls(LP.config(s))]


@pytest.mark.parametrize("shape, control", CONTROLS)
def test_negative_control_fails(cases, shape, control):
    """both references perturbed, the twin (standing in for the engine) not: the criterion must fail"""
    c = cases(shape)
    ctl = LP.controls(c["cfg"])[control]
    sd = ctl["edit"](c["sd"]) if ctl["edit"] else c["sd"]
    shift = ctl.get("shift_last", False)
    ref = torch.stack(LP.run_rows(LP.build_hf(c["cfg"], sd, torch.float64), c["seqs"], T, shift))
    hf = torch.stack(LP.run_rows(LP.build_hf(c["cfg"], sd, torch.bfloat16), c["seqs"], T, shift))
    r = LP.judge(c["twin"], hf, ref)
    caught = LP.logits_check_catches(c["twin"], hf, 1031, SEED)
    print(f"{shape} {control}: {LP.fmt(r)}; old logits check catches it: {caught}")
    assert not r["ok"], f"{control} not detected: {LP.fmt(r)}"
