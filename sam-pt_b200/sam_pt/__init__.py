"""Drop-in `sam_pt` package of the H100-native SAM-PT hot path (mirrors the dotted paths the reference's Hydra
configs target, SURVEY.md §8b).  Sub-packages are imported lazily: the reference's eager
`sam_pt/point_tracker/__init__.py:1-7` pulls in tensorflow/jax trackers that are out of scope here."""
