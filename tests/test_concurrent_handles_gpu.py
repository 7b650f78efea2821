"""GPU: distinct handles driven from distinct threads (include/jimm_b200.h: "a handle is not thread-safe, distinct handles are").

Each case runs in a fresh interpreter, so that no kernel of the library has been launched in it yet: the first forward of each GEMM /
attention variant sets its shared-memory attribute once per device, and four threads reach those first launches together.  The
outputs must be the bits of the same models run one at a time."""

import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def build_models():
    """Four small fp16 models whose forwards share GEMM instantiations: ViT with head width 64, ViT with head width 80 (the
    dynamic-shared-memory attention), a MAP-pooled tower and CLIP.  Seeded, so every process builds the same weights."""
    from jimm_b200 import Rngs
    from jimm_b200.common.vit import VisionTransformerBase
    from jimm_b200.models import CLIP, VisionTransformer

    f16 = torch.float16
    return {
        "vit_d64": VisionTransformer(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=1024, hidden_size=256,
                                     dtype=f16, rngs=Rngs(1)),
        "vit_d80": VisionTransformer(num_classes=10, img_size=64, patch_size=16, num_layers=2, num_heads=4, mlp_dim=1280, hidden_size=320,
                                     dtype=f16, rngs=Rngs(2)),
        "map_tower": VisionTransformerBase(img_size=64, patch_size=16, in_channels=3, hidden_size=256, num_layers=2, num_heads=4, mlp_dim=1024,
                                           pooling_type="MAP", layernorm_epsilon=1e-6, dtype=f16, rngs=Rngs(3)),
        "clip": CLIP(64, 2, 128, 16, 20, 300, 64, 1, 2, dtype=f16),
    }


def inputs():
    g = torch.Generator().manual_seed(5)
    img = torch.randn(3, 64, 64, 3, generator=g)
    ids = torch.randint(1, 300, (2, 20), generator=g, dtype=torch.int32)
    return img, ids


def run_one(name, n, img, ids):
    """One forward of handle n on the current stream; outputs on the device."""
    if name == "clip":
        return [n.vision(img, encode=True), n.text(ids)]
    return [n.vision(img)]


def handles(models):
    return {k: m.set_max_batch(4).native(4) for k, m in models.items()}


def _child(script, tmp_path, timeout=600):
    out = tmp_path / "out.pt"
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_concurrent_handles_gpu as T; T.{script}({str(out)!r})"
    r = subprocess.run([sys.executable, "-u", "-X", "faulthandler", "-c", code], capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    assert r.returncode == 0, f"child failed (exit {r.returncode}):\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}"
    print(r.stdout)
    return torch.load(out)


# ------------------------------------------------------------------------------------------------- first forwards from four threads
def first_forwards_from_threads(out_path):
    import threading

    torch.cuda.set_device(0)
    ns = handles(build_models())
    img, ids = inputs()
    img, ids = img.cuda(), ids.cuda()
    torch.cuda.synchronize()
    barrier = threading.Barrier(len(ns))
    results, errors = {}, {}

    def work(name):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                barrier.wait()  # ctypes releases the GIL: the four first forwards are enqueued at the same moment
                outs = run_one(name, ns[name], img, ids)
            s.synchronize()
            results[name] = [o.cpu() for o in outs]
        except Exception as e:  # noqa: BLE001  (reported to the parent)
            errors[name] = repr(e)

    ts = [threading.Thread(target=work, args=(k,)) for k in ns]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for n in ns.values():
        n.close()
    torch.save({"results": results, "errors": errors}, out_path)


def test_first_forwards_of_four_handles_from_four_threads(tmp_path):
    got = _child("first_forwards_from_threads", tmp_path)
    assert not got["errors"], got["errors"]
    img, ids = inputs()
    ns = handles(build_models())
    for name, n in ns.items():
        want = [o.cpu() for o in run_one(name, n, img.cuda(), ids.cuda())]
        for a, b in zip(got["results"][name], want):
            assert torch.equal(a, b), f"{name}: threaded first forward differs from the same model run alone"
        n.close()


# ------------------------------------------------------------------------------------- a load and a destroy beside graph replay
def load_beside_graph_replay(out_path):
    import threading

    from jimm_b200 import Rngs, _lib
    from jimm_b200.models import VisionTransformer

    torch.cuda.set_device(0)
    lib = _lib.load()
    models = build_models()
    serve = models["vit_d64"].set_max_batch(32).native(32)
    other = models["vit_d80"].set_max_batch(4).native(4)  # destroyed while `serve` replays
    big = VisionTransformer(num_classes=10, img_size=224, patch_size=16, num_layers=4, dtype=torch.float16, rngs=Rngs(7)).set_max_batch(2)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(32, 64, 64, 3, generator=g).cuda()
    xb = torch.randn(2, 224, 224, 3, generator=g).cuda()
    sizes = list(range(1, 33))
    want = {b: serve.vision(x[:b].contiguous()).cpu() for b in sizes}  # eager: every batch size's first call
    torch.cuda.synchronize()
    r0 = lib.jimm_graph_replay_count()
    barrier = threading.Barrier(2)
    done = threading.Event()
    res = {"mismatch": [], "errors": [], "serve_calls": 0}

    def serving():
        try:
            s = torch.cuda.Stream()
            barrier.wait()
            with torch.cuda.stream(s):
                while not done.is_set() or res["serve_calls"] < 2 * len(sizes):
                    b = sizes[res["serve_calls"] % len(sizes)]
                    o = serve.vision(x[:b].contiguous())  # second call of a size: captured; later calls: replayed
                    s.synchronize()
                    if not torch.equal(o.cpu(), want[b]):
                        res["mismatch"].append(b)
                    res["serve_calls"] += 1
        except Exception as e:  # noqa: BLE001
            res["errors"].append("serving: " + repr(e))

    def loading():
        try:
            barrier.wait()
            n = big.native(2)  # finalize: pinned staging, chunked packing, synchronisation
            res["loaded"] = n.vision(xb).cpu()
            other.close()
        except Exception as e:  # noqa: BLE001
            res["errors"].append("loading: " + repr(e))
        finally:
            done.set()

    ts = [threading.Thread(target=serving), threading.Thread(target=loading)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    res["replays"] = lib.jimm_graph_replay_count() - r0
    print(f"serving calls {res['serve_calls']}, graph replays {res['replays']}, errors {res['errors']}")
    serve.close()
    big.native(2).close()
    torch.save(res, out_path)


def test_load_and_destroy_beside_graph_replay(tmp_path):
    """One thread finalizes a new handle (then runs it, then destroys a third handle) while another replays small-batch CUDA graphs
    of its own handle: the load succeeds, the serving outputs keep their bits whether or not graph replay survives, and the loaded
    model computes what it computes alone."""
    from jimm_b200 import Rngs
    from jimm_b200.models import VisionTransformer

    got = _child("load_beside_graph_replay", tmp_path)
    assert not got["errors"], got["errors"]
    assert not got["mismatch"], f"serving outputs changed for batch sizes {sorted(set(got['mismatch']))}"
    print(f"graph replays during the load: {got['replays']} of {got['serve_calls']} serving calls")
    big = VisionTransformer(num_classes=10, img_size=224, patch_size=16, num_layers=4, dtype=torch.float16, rngs=Rngs(7)).set_max_batch(2)
    g = torch.Generator().manual_seed(8)
    torch.randn(32, 64, 64, 3, generator=g)
    xb = torch.randn(2, 224, 224, 3, generator=g).cuda()
    assert torch.equal(big(xb).cpu(), got["loaded"])
