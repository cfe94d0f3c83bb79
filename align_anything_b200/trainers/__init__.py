"""Hot-path mirrors of align_anything/trainers/<modality>/{dpo,ppo}.py: the same class and method
names, the same attributes read from `self`, the arithmetic on the sm_90a kernels.  Orchestration
(dataloaders, DeepSpeed engine init, generation, saving) is out of scope and stays in the reference;
`align_anything_b200.patch.install()` grafts these methods onto the reference classes."""
