"""Drivers of the offline-encoder protocol (AOTEngine.offline_encoder, then add_reference_frame / match_propogate_one_frame
without images), shaped like oracle.aot_oracle.run_video / run_video_events so a test can compare both paths frame by frame."""
import torch
import torch.nn.functional as F


def clip_masks(first_mask, T, events=None):
    """[T,1,H,W] label maps: the first-frame mask at step 0, `events` {step: [1,1,H,W]} at their steps, zeros elsewhere."""
    m = torch.zeros((T,) + tuple(first_mask.shape[1:]), dtype=torch.float32, device=first_mask.device)
    m[0] = first_mask[0]
    for t, v in (events or {}).items():
        m[t] = v[0].to(m.device, m.dtype)
    return m


def run_video_offline(engine, frames, first_mask, obj_num, output_size, forced_masks=None, stored_masks=True):
    """run_video on the offline path: the whole clip goes through offline_encoder first; the reference frame takes its mask
    from the stored masks (stored_masks) or from the argument.  Returns (low-res logits, output-size labels)."""
    engine.restart_engine()
    clip = torch.cat(list(frames), dim=0)
    engine.offline_encoder(clip, clip_masks(first_mask, len(frames)) if stored_masks else None)
    if stored_masks:
        engine.add_reference_frame(obj_nums=[obj_num], frame_step=0)
    else:
        engine.add_reference_frame(mask=first_mask, obj_nums=[obj_num], frame_step=0)
    logits_lo, labels = [], []
    for t in range(1, len(frames)):
        engine.match_propogate_one_frame()
        logit = engine.decode_current_logits(output_size)
        label = torch.argmax(torch.softmax(logit, dim=1), dim=1, keepdim=True).to(logit.dtype)
        lo = getattr(engine, "pred_id_logits", None)
        if lo is None and hasattr(engine, "aot_engines"):
            lo = engine.aot_engines[0].pred_id_logits
        logits_lo.append(lo.detach().clone())
        labels.append(label.detach().clone())
        fb = label if forced_masks is None else forced_masks[t - 1].to(label.device, label.dtype)
        engine.update_memory(F.interpolate(fb, size=tuple(engine.input_size_2d), mode="nearest"))
    return logits_lo, labels


def run_video_events_offline(engine, frames, first_mask, obj_num, output_size, new_objects, forced_masks):
    """run_video_events (teacher-forced) on the offline path: new objects are added as reference frames at their steps,
    with the fed-back label as the mask and no image."""
    engine.restart_engine()
    engine.offline_encoder(torch.cat(list(frames), dim=0))
    engine.add_reference_frame(mask=first_mask, obj_nums=[obj_num], frame_step=0)
    logits = []
    for t in range(1, len(frames)):
        engine.match_propogate_one_frame()
        logit = engine.decode_current_logits(output_size)
        label = forced_masks[t - 1].to(logit.device, logit.dtype)
        fb = F.interpolate(label, size=tuple(engine.input_size_2d), mode="nearest")
        new = new_objects.get(t)
        if new is not None:
            obj_num = max(obj_num, int(new.max().item()))
            engine.add_reference_frame(mask=fb, obj_nums=[obj_num], frame_step=t)
            logit = engine.decode_current_logits(output_size)
        engine.update_memory(fb)
        logits.append(logit.detach().clone())
    return logits
