"""Host-side (Python) cost of one training step: cProfile over a few PSPNet50 steps, top functions by own time and by
cumulative time. Run on a GPU box; kernels are asynchronous, so this is enqueue cost, not GPU time."""
import cProfile
import io
import os
import pstats
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from semseg_b200.pspnet import PSPNet  # noqa: E402


def main():
    torch.manual_seed(0)
    model = PSPNet(layers=50, classes=150, zoom_factor=8, pretrained=False).cuda().train()
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((16, 3, 473, 473), device="cuda", generator=g)
    y = torch.randint(0, 150, (16, 473, 473), device="cuda", generator=g)

    def step():
        _, ml, al = model(x, y)
        loss = ml + 0.4 * al
        opt.zero_grad()
        loss.backward()
        opt.step()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    pr = cProfile.Profile()
    pr.enable()
    for _ in range(5):
        step()
    pr.disable()
    torch.cuda.synchronize()
    out = io.StringIO()
    st = pstats.Stats(pr, stream=out)
    st.sort_stats("tottime").print_stats(35)
    st.sort_stats("cumulative").print_stats(45)
    txt = out.getvalue()
    os.makedirs(os.path.join(ROOT, "profile_out"), exist_ok=True)
    open(os.path.join(ROOT, "profile_out", "profile_cpu.txt"), "w").write(txt)
    print(txt[:6000])


if __name__ == "__main__":
    main()
