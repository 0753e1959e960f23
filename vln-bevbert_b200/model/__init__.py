"""The reference's model class surface (pretrain_src/model/{vilmodel,pretrain_cmt,bev_utils,ops}.py) on the
H100 kernels: same class names, constructor / forward signatures and state_dict keys."""
