"""Phase timing of the wgmma GEMM (debug %globaltimer stamps) for the decode shapes at R rows."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from llamagen_b200 import _lib
from util import test_gemm as run_gemm
os.environ["LG_GEMM_TC"] = "1"
lib = _lib.load()
lib.lg_debug_set_tc_trace.argtypes = [ctypes.c_void_p]
R = int(sys.argv[1]) if len(sys.argv) > 1 else 128
names = ["entry->setup", "setup->tma_issued", "setup->first_full", "first_full->last_full", "last_full->tmem_full", "tmem_full->stored", "stored->exit", "total"]
for (N, K, tag) in ((3072, 1024, "qkv"), (1024, 1024, "wo"), (5632, 1024, "w13"), (1024, 2816, "w2"), (16384, 1024, "head")):
    x = (torch.randn(R, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    for _ in range(3):
        run_gemm(x, w)
    trace = torch.zeros(4096 * 8, dtype=torch.int64, device="cuda")
    lib.lg_debug_set_tc_trace(ctypes.c_void_p(trace.data_ptr()))
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    run_gemm(x, w)
    ev1.record()
    torch.cuda.synchronize()
    lib.lg_debug_set_tc_trace(ctypes.c_void_p(0))
    t = trace.view(-1, 8).cpu()
    t = t[t[:, 0] > 0].double()
    g0 = t[:, 0].min()
    d = {"entry->setup": t[:, 1] - t[:, 0], "setup->tma_issued": t[:, 2] - t[:, 1], "setup->first_full": t[:, 3] - t[:, 1],
         "first_full->last_full": t[:, 4] - t[:, 3], "last_full->tmem_full": t[:, 5] - t[:, 4], "tmem_full->stored": t[:, 6] - t[:, 5],
         "stored->exit": t[:, 7] - t[:, 6], "total": t[:, 7] - t[:, 0]}
    print(f"{tag} N={N} K={K} R={R} ctas={t.shape[0]} stages_env={os.environ.get('LG_TC_STAGES')} kernel_span_ns={float(t[:,7].max()-g0):.0f} "
          f"first_entry_spread_ns={float(t[:,0].max()-g0):.0f} event_ms(gemm+reduce)={ev0.elapsed_time(ev1):.4f}")
    print("   " + "  ".join(f"{k}: {float(v.mean()):.0f}/{float(v.max()):.0f}" for k, v in d.items()))
