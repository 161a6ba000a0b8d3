"""Where does the end-to-end fp16 error come from?  (test infrastructure: uses the CPU oracle; run by hand, ~2 min)

    python tests/precision_study.py

Re-runs the oracle's SD1.5 + ControlNet rank-128 apply_model (B = 1, the golden-fixture inputs) in fp32 arithmetic with
fp16 ROUNDING inserted at the points where the CUDA path stores or feeds fp16: GEMM / conv operands (activations and
LoRA-folded weights), op outputs, attention probabilities, and the residual-stream sums.  Results (recorded in
the comments of tests/tolerances.py):
    all roundings (what the product does)      1.57e-3
    fp32 residual stream, fp16 operands        1.40e-3
    fp16 residual stream only                  0.98e-3
    only the weights rounded to fp16           0.88e-3
    only the activations rounded to fp16       1.10e-3
i.e. rounding the tensor-core OPERANDS to fp16 alone costs 1.4e-3 on this random-init network; the accumulated
residual-stream rounding adds 11 %.  An fp32 residual stream would not bring the end-to-end figure under 1e-3.
"""
import os, sys, time
import torch, torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ctrlora_oracle as O, synth
torch.set_num_threads(32)
g = torch.load(os.path.join(ROOT, 'tests', 'golden', 'sd15_rank128_golden.pt'), weights_only=False)
seed = g['seed']
s = synth.synth_state_dict(g['control_shapes'], seed, 'control_model.')
u = synth.synth_state_dict(g['unet_shapes'], seed, 'model.diffusion_model.')
sd = {'control_model.' + k: v for k, v in s.items()}
sd.update({'model.diffusion_model.' + k: v for k, v in u.items()})
x = synth.synth_input('x', (1, 4, 64, 64), seed); hint = synth.synth_input('hint', (1, 4, 64, 64), seed)
ctx = synth.synth_input('ctx', (1, 77, 768), seed); t = g['t']
rel = lambda a, b: ((a.float() - b.float()).norm() / b.float().norm()).item()
q = lambda z: z.half().float()

MODE = {'res': True, 'ops': True, 'w': True, 'a': True}
qw = lambda z: q(z) if MODE['w'] else z
qa = lambda z: q(z) if MODE['a'] else z   # res: round the residual sums to fp16; ops: round operands / op outputs to fp16
RESID_OUT = ('.out_layers.3', '.skip_connection', '.to_out.0', '.net.2', '.proj_out')

def linear(sd_, p, x_, lora_scale=1.0):
    W = sd_[p + '.weight']
    dk = p + '.lora_layer.down.weight'
    if dk in sd_:
        W = W + lora_scale * sd_[p + '.lora_layer.up.weight'] @ sd_[dk]     # folded like the product
    if MODE['ops']:
        y = F.linear(qa(x_), qw(W), sd_.get(p + '.bias'))
        return y if p.endswith(RESID_OUT) else qa(y)
    return F.linear(x_, W, sd_.get(p + '.bias'))

def conv(sd_, p, x_, stride=1, padding=0):
    if MODE['ops']:
        y = F.conv2d(qa(x_), qw(sd_[p + '.weight']), sd_.get(p + '.bias'), stride=stride, padding=padding)
        return y if p.endswith(RESID_OUT) else qa(y)
    return F.conv2d(x_, sd_[p + '.weight'], sd_.get(p + '.bias'), stride=stride, padding=padding)

def group_norm(sd_, p, x_, eps):
    y = F.group_norm((qa(x_) if MODE['ops'] else x_).float(), 32, sd_[p + '.weight'], sd_[p + '.bias'], eps)
    return y   # SiLU follows; rounding happens at the conv operand

def layer_norm(sd_, p, x_):
    return F.layer_norm(qa(x_) if MODE['ops'] else x_, (x_.shape[-1],), sd_[p + '.weight'], sd_[p + '.bias'], 1e-5)

def rq(z):
    return q(z) if MODE['res'] else z

def res_block(sd_, p, x_, emb):
    h = conv(sd_, p + '.in_layers.2', F.silu(group_norm(sd_, p + '.in_layers.0', x_, 1e-5)), padding=1)
    # the product adds the emb term inside the conv epilogue (fp32) before the fp16 store
    We = sd_[p + '.emb_layers.1.weight']
    if (p + '.emb_layers.1.lora_layer.down.weight') in sd_:
        We = We + sd_[p + '.emb_layers.1.lora_layer.up.weight'] @ sd_[p + '.emb_layers.1.lora_layer.down.weight']
    emb_out = F.linear(F.silu(emb), We, sd_[p + '.emb_layers.1.bias'])
    h = h + emb_out[:, :, None, None]
    h = conv(sd_, p + '.out_layers.3', F.silu(group_norm(sd_, p + '.out_layers.0', h, 1e-5)), padding=1)
    skip = conv(sd_, p + '.skip_connection', x_) if (p + '.skip_connection.weight') in sd_ else x_
    return rq(skip + h)

def cross_attention(sd_, p, x_, context, heads):
    c_ = x_ if context is None else context
    qq, k, v = linear(sd_, p + '.to_q', x_), linear(sd_, p + '.to_k', c_), linear(sd_, p + '.to_v', c_)
    b, n, c = qq.shape; d = c // heads
    split = lambda t_: t_.view(b, t_.shape[1], heads, d).permute(0, 2, 1, 3)
    qq, k, v = split(qq), split(k), split(v)
    sim = torch.einsum('bhid,bhjd->bhij', qq, k) * (d ** -0.5)
    pr = sim.softmax(dim=-1)
    if MODE['ops']:
        pr = qa(pr)
    out = torch.einsum('bhij,bhjd->bhid', pr, v)
    out = out.permute(0, 2, 1, 3).reshape(b, n, c)
    if MODE['ops']:
        out = qa(out)
    return linear(sd_, p + '.to_out.0', out)

def feed_forward(sd_, p, x_):
    W = sd_[p + '.net.0.proj.weight']; bb = sd_[p + '.net.0.proj.bias']
    dk = p + '.net.0.proj.lora_layer.down.weight'
    if dk in sd_:
        W = W + sd_[p + '.net.0.proj.lora_layer.up.weight'] @ sd_[dk]
    y = F.linear(qa(x_), qw(W), bb) if MODE['ops'] else F.linear(x_, W, bb)
    a, gate = y.chunk(2, dim=-1)
    hmid = a * F.gelu(gate)
    if MODE['ops']:
        hmid = qa(hmid)
    return linear(sd_, p + '.net.2', hmid)

def transformer_block(sd_, p, x_, context, heads):
    x_ = rq(cross_attention(sd_, p + '.attn1', layer_norm(sd_, p + '.norm1', x_), None, heads) + x_)
    x_ = rq(cross_attention(sd_, p + '.attn2', layer_norm(sd_, p + '.norm2', x_), context, heads) + x_)
    x_ = rq(feed_forward(sd_, p + '.ff', layer_norm(sd_, p + '.norm3', x_)) + x_)
    return x_

def spatial_transformer(sd_, p, x_, context, heads):
    b, c, h, w = x_.shape
    x_in = x_
    y = conv(sd_, p + '.proj_in', group_norm(sd_, p + '.norm', x_, 1e-6))
    y = y.permute(0, 2, 3, 1).reshape(b, h * w, -1)
    i = 0
    while (p + f'.transformer_blocks.{i}.norm1.weight') in sd_:
        y = transformer_block(sd_, p + f'.transformer_blocks.{i}', y, context, heads); i += 1
    y = y.reshape(b, h, w, -1).permute(0, 3, 1, 2)
    return rq(conv(sd_, p + '.proj_out', y) + x_in)

for name in ('linear', 'conv', 'group_norm', 'layer_norm', 'res_block', 'cross_attention', 'feed_forward', 'transformer_block', 'spatial_transformer'):
    setattr(O, name, globals()[name])

def run():
    with torch.no_grad():
        return O.apply_model(sd, x, t, ctx, hint, 8, 320)

t0 = time.time()
MODE.update(res=False, ops=False); ref = run(); print('fp32 vs reference golden', rel(ref, g['eps']), time.time() - t0)
MODE.update(res=True, ops=True, w=True, a=True); a = run(); print('A: fp16 ops + fp16 residual stream  :', rel(a, ref))
MODE.update(res=False, ops=True, w=True, a=True); b = run(); print('B: fp16 ops, fp32 residual stream   :', rel(b, ref))
MODE.update(res=True, ops=False, w=True, a=True); c = run(); print('C: fp32 ops, fp16 residual stream   :', rel(c, ref))
MODE.update(res=False, ops=True, w=True, a=False); d = run(); print('D: only weights rounded to fp16      :', rel(d, ref))
MODE.update(res=False, ops=True, w=False, a=True); e = run(); print('E: only activations rounded to fp16  :', rel(e, ref))
