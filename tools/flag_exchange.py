"""cycles per round of bare all-to-all flag exchanges among co-resident CTAs (tsb_debug_flag_exchange): what ordering
rounds with release / acquire fences costs, and how one exchange scales with the number of CTAs (the persistent
N-Queens kernel's CTA counts rest on it):
python tools/flag_exchange.py [variant[:ctas] ...]"""
import ctypes as C, sys
sys.path.insert(0, "gpu-accelerated-tree-search-chapel_b200")
import tsb200
L = tsb200.lib()
L.tsb_init_devices(1)
names = {1: "no-release-fence", 2: "no-acquire-fence", 4: "16B/thread stores", 8: "cg polls", 16: "one exchange only"}
runs = [tuple(int(x) for x in (a.split(":") + ["0"])[:2]) for a in sys.argv[1:]] or \
    [(0, 0), (3, 0), (16, 0), (16, 74), (16, 32), (16, 8), (16, 2), (3, 32), (3, 8), (0, 8)]
for variant, ctas in runs:
    out = C.c_double(0)
    for _ in range(2):
        rc = L.tsb_debug_flag_exchange(0, 20000, variant, ctas, C.byref(out))
    desc = ", ".join(v for b, v in names.items() if variant & b) or "two exchanges, release + acquire fences"
    print(f"variant {variant:2d} ctas {ctas or 'all':>3} ({desc}): rc={rc} {out.value:.0f} cycles per round", flush=True)
