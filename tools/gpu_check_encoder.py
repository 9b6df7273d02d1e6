"""First-light / regression check of the encoder kernels (GEMM, LayerNorm, attention, full forward) on an H100.

Each case runs in its own subprocess with a timeout.  Usage on the GPU box:
    python tools/gpu_check_encoder.py [--only gemm|attn|ln|enc|perf]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEMM_CASES = [  # M, N, K, epi
    (128, 128, 64, 0), (129, 256, 128, 0), (255, 128, 64, 2), (257, 384, 384, 1), (300, 384, 384, 0),
    (1000, 1152, 384, 0), (777, 1536, 384, 1), (512, 384, 1536, 2), (16384, 3072, 1024, 0), (16384, 1024, 1024, 2),
    (16384, 4096, 1024, 1), (16384, 1024, 4096, 2), (16384, 1152, 384, 0), (16384, 384, 1536, 2),
    (16384, 768, 3072, 2), (16384, 768, 768, 2), (1000, 1024, 384, 1),
]
ATTN_CASES = [  # H, heads, lengths, tc (1 = wgmma kernel)
    (128, 4, [5, 64, 65, 1, 130], 0), (1024, 16, [512, 33, 200, 512], 0), (384, 12, [77, 512, 300], 0), (768, 12, [128] * 6, 0),
    (128, 2, [5, 64, 65, 1, 130, 128, 129, 300], 1), (1024, 16, [512, 33, 200, 512], 1), (768, 12, [128] * 6, 1),
    (1024, 16, [512] * 32, 0), (1024, 16, [512] * 32, 1),
    (1024, 16, [37, 512, 100, 64, 63, 191, 192, 193], 1),
]
ENC_CASES = [  # name, cfg args, lengths, std
    ("tiny", (128, 2, 4, 256, 1000), [5, 64, 65, 1, 130, 17], 0.02),
    ("tiny-wide-init", (128, 2, 4, 256, 1000), [12, 40, 200], 0.08),
    ("small-4L", (384, 4, 12, 1536, 30522), [512, 100, 37, 256], 0.02),
    ("large-2L", (1024, 2, 16, 4096, 30522), [512, 333, 64], 0.02),
    ("large-24L", (1024, 24, 16, 4096, 30522), [512, 128, 300, 45], 0.02),
]


def gemm_case(i):
    import torch
    from comorag_b200 import _native
    lib = _native.load()
    M, N, K, epi = GEMM_CASES[i]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(i)
    a = (torch.randn(M, K, generator=g, device=dev) * 0.5).bfloat16()
    w = (torch.randn(N, K, generator=g, device=dev) * 0.05).bfloat16()
    bias = torch.randn(N, generator=g, device=dev)
    res = (torch.randn(M, N, generator=g, device=dev)).bfloat16()
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def run():
        rc = lib.crag_gemm_bf16(a.data_ptr(), K, w.data_ptr(), K, bias.data_ptr(), res.data_ptr(), N, out.data_ptr(), N,
                                M, N, K, epi, st)
        _native.check(rc, "crag_gemm_bf16")
    run()
    torch.cuda.synchronize()
    ref = a.float() @ w.float().T + bias
    if epi == 1:
        ref = torch.nn.functional.gelu(ref)
    if epi == 2:
        ref = ref + res.float()
    err = (out.float() - ref).abs()
    tol = 0.01 * ref.abs() + 0.02
    r = {"kind": "gemm", "shape": [M, N, K, epi], "max_err": float(err.max()), "ok": bool((err <= tol).all()),
         "bad_frac": float((err > tol).float().mean())}
    if M >= 4096:
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        r.update(ms=ms, tflops=2.0 * M * N * K / ms / 1e9)
    return r


def attn_case(i):
    import torch
    from comorag_b200 import _native
    lib = _native.load()
    H, heads, lens, tc = ATTN_CASES[i]
    dh = H // heads
    dev = torch.device("cuda:0")
    T = sum(lens)
    g = torch.Generator(device=dev).manual_seed(100 + i)
    qkv = (torch.randn(T, 3 * H, generator=g, device=dev)).bfloat16()
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
    ctx = torch.zeros(T, H, dtype=torch.bfloat16, device=dev)
    def run():
        if tc:
            rc = lib.crag_attention_varlen_tc(qkv.data_ptr(), cu.data_ptr(), len(lens), T, max(lens), H, heads | ((tc - 1) << 8), ctx.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream)
        else:
            rc = lib.crag_attention_varlen(qkv.data_ptr(), cu.data_ptr(), len(lens), max(lens), H, heads, ctx.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream)
        _native.check(rc, "crag_attention_varlen")
    run()
    torch.cuda.synchronize()
    ref = torch.zeros(T, H, device=dev)
    s = 0
    for L in lens:
        x = qkv[s:s + L].float()
        q, k, v = (x[:, j * H:(j + 1) * H].view(L, heads, dh).transpose(0, 1) for j in range(3))
        att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(dh), dim=-1)
        ref[s:s + L] = (att @ v).transpose(0, 1).reshape(L, H)
        s += L
    err = (ctx.float() - ref).abs()
    res = {"kind": "attn", "tc": tc, "shape": [H, heads, lens[:8], len(lens)], "max_err": float(err.max()), "ok": bool(err.max() < 0.03)}
    if T >= 8192:
        for _ in range(3):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 20
        res.update(ms=ms, tflops=sum(4.0 * L * L * dh * heads for L in lens) / ms / 1e9)
    return res


def ln_case(i):
    import torch
    from comorag_b200 import _native
    lib = _native.load()
    H = [128, 384, 768, 1024][i]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(i)
    x = (torch.randn(1001, H, generator=g, device=dev) * 3 + 1).bfloat16()
    gam, bet = torch.randn(H, generator=g, device=dev), torch.randn(H, generator=g, device=dev)
    out = torch.zeros_like(x)
    rc = lib.crag_layernorm(x.data_ptr(), 1001, H, gam.data_ptr(), bet.data_ptr(), 1e-12, out.data_ptr(),
                            torch.cuda.current_stream().cuda_stream)
    _native.check(rc, "crag_layernorm")
    ref = torch.nn.functional.layer_norm(x.float(), (H,), gam, bet, 1e-12)
    err = (out.float() - ref).abs()
    return {"kind": "ln", "H": H, "max_err": float(err.max()), "ok": bool((err <= 0.01 * ref.abs() + 0.01).all())}


def enc_case(i):
    import torch
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig, random_state_dict
    from oracle.encoder_oracle import encode_token_lists
    name, cargs, lens, std = ENC_CASES[i]
    cfg = EncoderConfig(*cargs)
    dev = torch.device("cuda:0")
    sd = random_state_dict(cfg, seed=i, std=std, device=dev)
    # the engine stores bf16 weights; give the oracle the same (bf16-rounded) weights so only arithmetic differs
    sd_q = {k: (v.bfloat16().float() if v.dim() == 2 else v) for k, v in sd.items()}
    enc = BertEncoderB200(cfg, sd, dev)
    g = torch.Generator().manual_seed(7)
    seqs = [[101] + torch.randint(1000 if cfg.vocab_size > 2000 else 5, cfg.vocab_size, (L - 2,), generator=g).tolist() + [102]
            if L >= 2 else [101] for L in lens]
    out = enc.encode_token_lists(seqs)
    torch.cuda.synchronize()
    ref = encode_token_lists(sd_q, cfg, seqs)
    ref_fp32w = encode_token_lists(sd, cfg, seqs)
    cos = torch.nn.functional.cosine_similarity(out, ref, dim=1)
    cos2 = torch.nn.functional.cosine_similarity(out, ref_fp32w, dim=1)
    maxabs = float((out - ref).abs().max())
    return {"kind": "enc", "name": name, "min_cos_vs_bf16w": float(cos.min()), "min_cos_vs_fp32w": float(cos2.min()),
            "max_abs": maxabs, "max_abs_fp32w": float((out - ref_fp32w).abs().max()),
            "norms": [float(x) for x in out.norm(dim=1)[:3]],
            "pair_cos_ref": float(torch.nn.functional.cosine_similarity(ref[0], ref[1], dim=0)) if len(lens) > 1 else None,
            "ok": bool(cos.min() > 0.999 and maxabs < 1e-2)}


def perf_case(i):
    import torch
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig
    shapes = [("bge-large", EncoderConfig.bge_large()), ("bge-small", EncoderConfig.bge_small()), ("bge-base", EncoderConfig.bge_base())]
    name, cfg = shapes[i]
    dev = torch.device("cuda:0")
    enc = BertEncoderB200.random_init(cfg, 0, device=dev)
    n, L = 32, 512
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(1000, cfg.vocab_size, (n * L,), generator=g, dtype=torch.int32).to(dev)
    cu = (torch.arange(n + 1, dtype=torch.int32) * L).to(dev)
    out = torch.empty(n, cfg.hidden_size, device=dev)
    for _ in range(3):
        enc.forward_packed(ids, cu, L, out_f32=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5
    e0.record()
    for _ in range(reps):
        enc.forward_packed(ids, cu, L, out_f32=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    fl = cfg.flops_per_chunk(L) * n
    return {"kind": "perf", "name": name, "ms_per_batch": ms, "chunks_per_s": n / ms * 1e3, "tflops": fl / ms / 1e9}


KINDS = {"gemm": (gemm_case, len(GEMM_CASES)), "ln": (ln_case, 4), "attn": (attn_case, len(ATTN_CASES)),
         "enc": (enc_case, len(ENC_CASES)), "perf": (perf_case, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", default=None)
    ap.add_argument("--case", type=int, default=None)
    ap.add_argument("--only", default=None)
    ap.add_argument("--timeout", type=int, default=300)
    args = ap.parse_args()
    if args.kind is not None:
        print("RESULT " + json.dumps(KINDS[args.kind][0](args.case)))
        return
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    results = []
    for kind, (_, n) in KINDS.items():
        if args.only and kind not in args.only.split(","):
            continue
        for i in range(n):
            try:
                p = subprocess.run([sys.executable, __file__, "--kind", kind, "--case", str(i)], capture_output=True,
                                   text=True, timeout=args.timeout)
                line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
                r = json.loads(line[-1][7:]) if line else {"kind": kind, "case": i, "ok": False, "rc": p.returncode,
                                                            "stderr": p.stderr[-1200:]}
            except subprocess.TimeoutExpired:
                r = {"kind": kind, "case": i, "ok": False, "error": "timeout"}
            results.append(r)
            print(json.dumps(r), flush=True)
    with open(os.path.join(ROOT, "gpurun_out", "check_encoder.json"), "w") as f:
        json.dump(results, f, indent=1)
    print("SUMMARY", sum(1 for r in results if r.get("ok", True)), "/", len(results), "ok")


if __name__ == "__main__":
    main()
