"""Large-image searches with the full-size model (BASELINE.json configs[2..4] shapes): node counts, crops/s, memory."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from PIL import Image
from vstar_b200 import synth
from vstar_b200.config import VSMConfig
from vstar_b200.engine import VSMEngine, VSMWeights
from vstar_b200.visual_search import visual_search
from vstar_b200.vsm import VSM

cfg = VSMConfig()
shapes = synth.state_dict_shapes(cfg)
eng = VSMEngine(VSMWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=1234, device="cuda")), max_tokens=384)
prompt, ans = synth.synthetic_prompt(cfg, n_text=60, seed=0, im_start_index=37)


class V(VSM):
    def _ids(self, q):
        return prompt[0].tolist()


vsm = V(engine=eng, forced_answer_ids=ans.tolist(), frontier_batch=64)
kw = dict(confidence_high=2.0, target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9)
out = []
for size, smallest, expect in [(2048, 512, 21), (4096, 512, 85), (8192, 1024, 85), (8192, 256, 1365)]:
    r = None
    for rep in range(2):              # rep 0 pays the one-time costs of new sizes (coefficient tables, allocator growth, pinning)
        img = Image.fromarray(np.random.default_rng(size + rep).integers(0, 256, (size, size, 3), dtype=np.uint8), "RGB")
        torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        fs, pl, ok, av, st = visual_search(vsm, img, "mug", None, smallest, batch_size=64, return_state=True, **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        vsm.release()
        assert len(st.search_path) == expect, (size, smallest, len(st.search_path))
        if rep == 0:
            first = dt
        else:
            r = dict(image=size, smallest=smallest, nodes=len(st.search_path), evals=st.n_evals, expect=expect, seconds_first_run=round(first, 3),
                     seconds=round(dt, 3), crops_per_s=round(st.n_evals / dt, 1), peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 1))
            print(json.dumps(r), flush=True)
        for node in st.search_path:
            node.pop("_heat", None); node.pop("final_heatmap", None)
        del st
        torch.cuda.empty_cache()
        if size == 8192 and smallest == 256 and rep == 0:
            pass
    out.append(r)
os.makedirs("bench_out", exist_ok=True)
json.dump(out, open("bench_out/big_search.json", "w"), indent=1)
