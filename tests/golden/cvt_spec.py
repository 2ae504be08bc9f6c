"""CvT parity cases (reference cvt.py), on the shared recipe of parity.py.  Its own rule, LeViT's: every BatchNorm's
weight, bias, running mean and running variance are perturbed (the default statistics would leave the BatchNorm folds
of the convolutional projections untested) and the statistics rounded to bf16 like the parameters."""
from levit_spec import perturb_batchnorms
from parity import Family

# every Transformer runs heads of 64 (the reference never passes dim_head down)
SMALL = dict(num_classes=7, s1_emb_dim=16, s1_heads=2, s2_emb_dim=32, s2_heads=2, s2_depth=1, s3_emb_dim=48,
             s3_heads=2, s3_depth=2)
BATCH = 2
# constructor keywords (on top of SMALL unless `readme`); `input` = (height, width) of the image, `batch` its batch
# size.  The comments give per stage the query map -> the key / value map.
CVT_CASES = {
    # the README config at 224, batch 1: 56 x 56 -> 28 x 28 (784 keys, more than attention_kv keeps in shared memory
    # at dim_head 64), 28 x 28 -> 14 x 14, 14 x 14 -> 7 x 7; stage 3 has 4 heads (256 wide) at dim 384
    "readme_224": dict(seed=701, readme=True, num_classes=1000, s1_emb_dim=64, s1_emb_kernel=7, s1_emb_stride=4,
                       s1_proj_kernel=3, s1_kv_proj_stride=2, s1_heads=1, s1_depth=1, s1_mlp_mult=4, s2_emb_dim=192,
                       s2_emb_kernel=3, s2_emb_stride=2, s2_proj_kernel=3, s2_kv_proj_stride=2, s2_heads=3, s2_depth=2,
                       s2_mlp_mult=4, s3_emb_dim=384, s3_emb_kernel=3, s3_emb_stride=2, s3_proj_kernel=3,
                       s3_kv_proj_stride=2, s3_heads=4, s3_depth=10, s3_mlp_mult=4, dropout=0., input=(224, 224),
                       batch=1),
    # odd and non-square maps, one channel: 25 x 19 -> 13 x 10, 13 x 10 -> 7 x 5, 7 x 5 -> 4 x 3
    "odd_nonsquare_c1": dict(seed=702, channels=1, input=(100, 75)),
    # other projection kernels and strides: 16 x 16 (k 1, s 1) -> 16 x 16, 8 x 8 (k 5, s 3) -> 3 x 3, 4 x 4 (k 7,
    # s 2: every tap of a key reaches past the map) -> 2 x 2
    "proj_kernels": dict(seed=703, s1_proj_kernel=1, s1_kv_proj_stride=1, s2_proj_kernel=5, s2_kv_proj_stride=3,
                         s3_proj_kernel=7, input=(64, 64)),
    # an even embedding kernel, which the reference accepts: k 4, stride 4, padding 2: 17 x 17 -> 9 x 9, 9 x 9 -> 5 x 5,
    # 5 x 5 -> 3 x 3
    "even_emb_kernel": dict(seed=704, s1_emb_kernel=4, s1_emb_stride=4, input=(64, 64)),
    # a tiny image: 4 x 4 -> 2 x 2, 2 x 2 -> 1 x 1, 1 x 1 -> 1 x 1 (one key)
    "tiny_16": dict(seed=705, input=(16, 16)),
    # mlp_mult 2, dropout 0.1 (eval), stride 3 keys at stage 1, batch 3: 12 x 20 -> 4 x 7, 6 x 10 -> 3 x 5, 3 x 5 ->
    # 2 x 3
    "mlp2_dropout_b3": dict(seed=706, s1_mlp_mult=2, s2_mlp_mult=2, s3_mlp_mult=2, s1_kv_proj_stride=3, dropout=0.1,
                            input=(48, 80), batch=3),
}
# the seeded-init (unperturbed) comparison
INIT_SEED = 721
INIT_KWARGS = dict(SMALL, s2_depth=2)

_SPEC_KEYS = ("seed", "input", "batch", "readme")


def case_kwargs(spec: dict) -> dict:
    kw = {} if spec.get("readme") else dict(SMALL)
    kw.update({k: v for k, v in spec.items() if k not in _SPEC_KEYS})
    return kw


def input_shape(spec: dict) -> tuple:
    return (spec.get("batch", BATCH), spec.get("channels", 3), *spec["input"])


FAMILY = Family(
    name="cvt", model="cvt.CvT", cases=CVT_CASES, case_kwargs=case_kwargs, input_shape=input_shape,
    init_seed=INIT_SEED, init={None: INIT_KWARGS}, after=perturb_batchnorms)
