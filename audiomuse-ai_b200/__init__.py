"""audiomuse-ai_b200: H100-native (sm_90a) replacement for AudioMuse-AI's CLAP analysis hot
path and its downstream k-NN / k-means, behind the reference's own Python call surface.

Import name: ``audiomuse_ai_b200`` (see the loader stub ``audiomuse_ai_b200.py`` at the repo
root; the directory keeps the hyphenated project name).

    clap_analyzer     -> tasks/clap_analyzer.py  (compute_mel_spectrogram, analyze_audio_file, ...)
    voyager_compat    -> the voyager.Index duck type used by tasks/voyager_manager.py and
                         tasks/clap_text_search.py
    clustering_gpu    -> tasks/clustering_gpu.py (GPUKMeans, get_clustering_model)
    dist              -> one-process-per-GPU sharding (torch.distributed / NCCL plumbing)

Nothing here touches CUDA at import time.
"""
__version__ = "0.1.0"
