"""MobileSAM (ChaoningZhang/MobileSAM) as the reference's YAML names it: TinyViT image encoder, SAM's prompt encoder and
mask decoder (configs/model/sam/sam_mobile_vit_tiny.yaml).  The encoder runs in libsampt_b200 (csrc/tinyvit.cu)."""
