"""GPU triage ladder: runs every kernel-vs-oracle check in its own subprocess (a device trap in one
check cannot poison the next), first on the wgmma product path and -- for triage only -- on the debug
SIMT GEMM backend (NEWSREC_DEBUG_SIMT_GEMM=1, same epilogue functors).  Writes gpurun_out/ladder.json.

    python tools/gpu_ladder.py            # everything
    python tools/gpu_ladder.py --only linear_small,nrms_golden
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "news-recommendation_b200", "src")):
    if p not in sys.path:
        sys.path.insert(0, p)

CHECKS = {
    "prep_gather": ("check_prep_and_gather", {}),
    "linear_tiny": ("check_linear", dict(M=128, N=64, K=64)),
    "linear_k300": ("check_linear", dict(M=128, N=200, K=300)),
    "linear_small": ("check_linear", dict(M=300, N=900, K=300)),
    "linear_multi_tile": ("check_linear", dict(M=128 * 9 + 17, N=900, K=300)),
    "linear_k900": ("check_linear", dict(M=777, N=300, K=900, out_bf16=0)),
    "linear_big": ("check_linear", dict(M=128 * 600 + 5, N=900, K=300)),
    "linear_conv3": ("check_linear", dict(M=37, N=300, K=300, taps=3, seg=20, relu=1)),
    "linear_conv3_f400_t50": ("check_linear", dict(M=11, N=400, K=300, taps=3, seg=50, relu=1)),
    "gemm_tn_small": ("check_gemm_tn", dict(Kr=64, Ma=128, Nb=64)),
    "gemm_tn": ("check_gemm_tn", dict(Kr=1000, Ma=900, Nb=301)),
    "gemm_tn_long": ("check_gemm_tn", dict(Kr=64 * 700 + 13, Ma=200, Nb=301)),
    "gemm_tn_shift": ("check_gemm_tn", dict(Kr=900, Ma=300, Nb=301, shift=1)),
    "gemm_tn_shift_neg": ("check_gemm_tn", dict(Kr=900, Ma=400, Nb=301, shift=-1)),
    "mhsa_core_t20": ("check_mhsa_core", dict(n_seq=7, T=20)),
    "mhsa_core_t50": ("check_mhsa_core", dict(n_seq=3, T=50)),
    "mhsa_core_many": ("check_mhsa_core", dict(n_seq=2000, T=20)),
    "mhsa_core_t16_dk10": ("check_mhsa_core", dict(n_seq=5, T=16, heads=30, dk=10)),
    "mhsa_core_t33_dk15": ("check_mhsa_core", dict(n_seq=5, T=33, heads=20, dk=15)),
    "mhsa_core_t64_dk30": ("check_mhsa_core", dict(n_seq=4, T=64, heads=10, dk=30)),
    "mhsa_core_t7_dk25": ("check_mhsa_core", dict(n_seq=9, T=7, heads=12, dk=25)),
    "additive": ("check_additive", {}),
    "additive_s50": ("check_additive", dict(N=9, S=50)),
    "additive_s4_f400": ("check_additive", dict(N=50, S=4, D=400)),
    "backend_agreement": ("check_backend_agreement", {}),
    "backend_agreement_1tile": ("check_backend_agreement", dict(M=4000)),
    "encoder_backend_diff": ("check_encoder_backend_diff", {}),
    "dot_score": ("check_dot_score", {}),
    "nrms_golden": ("check_nrms_golden", {}),
    "golden_nrms": ("check_golden", dict(case="nrms")),
    "golden_naml": ("check_golden", dict(case="naml")),
    "golden_naml_f400": ("check_golden", dict(case="naml_f400")),
    "golden_tanr": ("check_golden", dict(case="tanr")),
    "golden_lstur_ini": ("check_golden", dict(case="lstur_ini")),
    "golden_lstur_con": ("check_golden", dict(case="lstur_con")),
    "nrms_random": ("check_nrms_random", {}),
    "nrms_eval_api": ("check_nrms_eval_api", {}),
    "nrms_train_mode": ("check_nrms_train_mode", {}),
    "nrms_full_size": ("check_nrms_full_size_properties", {}),
    "cnn_naml_title_full": ("check_cnn_encoder", dict(n_seq=512 * 55, T=20, d=300, F=400, q=200, V=70976, p_drop=0.2)),
    "cnn_naml_abstract": ("check_cnn_encoder", dict(n_seq=128 * 55, T=50, d=300, F=400, q=200, V=5000, p_drop=0.2)),
    "cnn_lstur_accurate": ("check_cnn_encoder", dict(n_seq=2000, T=20, d=300, F=300, q=200, V=3000, accurate=True)),
    "cnn_tanr_eval": ("check_cnn_encoder", dict(n_seq=2000, T=20, d=300, F=400, q=200, V=3000, p_drop=0.0)),
    "cnn_t1": ("check_cnn_encoder", dict(n_seq=999, T=1, d=300, F=300, q=200, V=3000)),
    "cnn_t64": ("check_cnn_encoder", dict(n_seq=97, T=64, d=300, F=300, q=200, V=3000)),
    "cnn_f8_q16": ("check_cnn_encoder", dict(n_seq=613, T=20, d=64, F=8, q=16, V=37, p_drop=0.5)),
    "element_encoder": ("check_element_encoder", dict(n=512 * 55, E=100, F=400)),
    "linear_rows_topic": ("check_linear_rows", dict(n=512 * 5, K=300, N=275, relu=1)),
    "linear_rows_k900": ("check_linear_rows", dict(n=777, K=900, N=300, relu=1, strided=True)),
    "embedding_f32": ("check_embedding_f32", dict(n=512 * 55, V=300, D=100)),
}


def run_one(name):
    import torch  # noqa: F401
    import gpu_checks
    fn, kw = CHECKS[name]
    t0 = time.time()
    res = getattr(gpu_checks, fn)(**kw)
    torch.cuda.synchronize()
    res["seconds"] = round(time.time() - t0, 2)
    print("RESULT " + json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--one")
    ap.add_argument("--only", default="")
    ap.add_argument("--skip-simt", action="store_true")
    ap.add_argument("--timeout", type=int, default=240)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "ladder.json"))
    a = ap.parse_args()
    if a.one:
        run_one(a.one)
        return
    names = [n for n in CHECKS if not a.only or n in a.only.split(",")]
    results = {}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    for backend in (["wgmma"] if a.skip_simt else ["wgmma", "simt_debug"]):
        for n in names:
            if backend == "simt_debug" and n in ("linear_big", "nrms_full_size", "gemm_tn_long"):
                continue
            env = dict(os.environ)
            env["NEWSREC_DEBUG_SIMT_GEMM"] = "1" if backend == "simt_debug" else "0"
            env["PYTHONHASHSEED"] = "0"
            t0 = time.time()
            try:
                pr = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", n], env=env, capture_output=True,
                                    text=True, timeout=a.timeout)
                line = [l for l in pr.stdout.splitlines() if l.startswith("RESULT ")]
                if pr.returncode == 0 and line:
                    res = json.loads(line[-1][7:])
                else:
                    res = {"error": (pr.stderr or pr.stdout)[-1500:], "returncode": pr.returncode}
            except subprocess.TimeoutExpired:
                res = {"error": "timeout"}
            res["wall"] = round(time.time() - t0, 1)
            results[f"{backend}:{n}"] = res
            print(f"[{backend}] {n}: {json.dumps(res)[:600]}", flush=True)
            with open(a.out, "w") as f:
                json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
