"""TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ -- never by the product path).

Plain-torch restatement of LPIPS v0.1 with the AlexNet backbone, as SplaTAM's evaluation calls it through torchmetrics
(LearnedPerceptualImagePatchSimilarity(net_type='alex', normalize=True) on clamp(weighted image, 0, 1),
R/utils/eval_helpers.py:484-485, 730-731); device-agnostic, float64 by default; the checker for csrc/lpips.cu.

  1. x <- 2x - 1, then (x - LPIPS_SHIFT) / LPIPS_SCALE per channel (the scaling layer)
  2. torchvision AlexNet features: f1 = relu(conv1) (11x11, stride 4, pad 2), max-pool 3x3/2, f2 = relu(conv2)
     (5x5, pad 2), max-pool 3x3/2, f3..f5 = relu(conv3..conv5) (3x3, pad 1)
  3. per layer and pixel: n = f / sqrt(LPIPS_EPS + sum_c f^2) for both images, d = sum_c lin_c (n_x - n_y)^2
  4. LPIPS = sum over the five layers of the mean of d over the layer's pixels

`weights` is one dict holding both state dicts as they are stored: torchvision's alexnet (features.{0,3,6,8,10}.weight
/ .bias) and lpips' alex.pth (lin{0..4}.model.1.weight, [1,C,1,1]).
"""
import torch
import torch.nn.functional as F

LPIPS_SHIFT = (-0.030, -0.088, -0.188)
LPIPS_SCALE = (0.458, 0.448, 0.450)
LPIPS_EPS = 1e-8                 # torchmetrics' normalisation: f / sqrt(eps + sum_c f^2)
# torchvision alexnet: (features index, Cin, Cout, kernel, stride, padding) of the five convolutions
ALEX_CONVS = ((0, 3, 64, 11, 4, 2), (3, 64, 192, 5, 1, 2), (6, 192, 384, 3, 1, 1), (8, 384, 256, 3, 1, 1),
              (10, 256, 256, 3, 1, 1))


def features(x, weights, dtype=torch.float64):
    """The five AlexNet feature maps f1..f5 of [N,3,H,W] images in [0,1] (clamped here), computed in `dtype`."""
    x = x.to(dtype).clamp(0, 1)
    shift = torch.tensor(LPIPS_SHIFT, dtype=dtype, device=x.device).reshape(1, 3, 1, 1)
    scale = torch.tensor(LPIPS_SCALE, dtype=dtype, device=x.device).reshape(1, 3, 1, 1)
    h = (2 * x - 1 - shift) / scale
    out = []
    for l, (idx, _, _, _, stride, pad) in enumerate(ALEX_CONVS):
        if l in (1, 2):
            h = F.max_pool2d(h, kernel_size=3, stride=2)
        w = weights["features.%d.weight" % idx].to(device=x.device, dtype=dtype)
        b = weights["features.%d.bias" % idx].to(device=x.device, dtype=dtype)
        h = torch.relu(F.conv2d(h, w, b, stride=stride, padding=pad))
        out.append(h)
    return out


def lpips(x, y, weights, dtype=torch.float64):
    """[N] LPIPS of the image pairs x[i], y[i] ([N,3,H,W]), computed in `dtype`."""
    total = 0
    for l, (fx, fy) in enumerate(zip(features(x, weights, dtype), features(y, weights, dtype))):
        nx = fx / torch.sqrt(LPIPS_EPS + (fx ** 2).sum(1, keepdim=True))
        ny = fy / torch.sqrt(LPIPS_EPS + (fy ** 2).sum(1, keepdim=True))
        lin = weights["lin%d.model.1.weight" % l].to(device=x.device, dtype=dtype)
        total = total + F.conv2d((nx - ny) ** 2, lin).mean(dim=(1, 2, 3))
    return total


def random_state_dicts(seed=0):
    """Seeded stand-ins for the two weight files in their real key layout: (alexnet state dict, lpips alex state dict).
    Conv weights at Kaiming scale, small positive biases (so the ReLUs are neither all on nor all off), non-negative
    linear heads; torchvision's classifier keys are included, as the real file has them."""
    g = torch.Generator().manual_seed(seed)
    alex, lin = {}, {}
    for l, (idx, cin, cout, k, _, _) in enumerate(ALEX_CONVS):
        alex["features.%d.weight" % idx] = torch.randn(cout, cin, k, k, generator=g) * (2.0 / (cin * k * k)) ** 0.5
        alex["features.%d.bias" % idx] = 0.05 * torch.rand(cout, generator=g)
        lin["lin%d.model.1.weight" % l] = torch.rand(1, cout, 1, 1, generator=g) / cout ** 0.5
    alex["classifier.1.weight"] = torch.randn(16, 8, generator=g)
    alex["classifier.1.bias"] = torch.zeros(16)
    return alex, lin
