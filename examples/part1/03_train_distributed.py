"""Part 1 / 03_model_training_distributed  (reference: 03_model_training_distributed.py) - the main path.

converter (sharded loader) -> `train_and_evaluate_hvd()` per rank -> Runner(np).run(...) -> rank 0 logs + returns.
On an 8xH100 box set HVD_NP=8: the gradient all-reduce inside DistributedOptimizer is our fused NVLS/P2P kernel."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from common import *  # noqa: F401,F403
from b200ddl import optim, tracking
from b200ddl import parallel as hvd
from b200ddl.loader import make_converter
from b200ddl.models import build_model
from b200ddl.parallel import Runner
from b200ddl.train import ReduceLROnPlateau, Trainer

BATCH_SIZE = int(os.environ.get("BATCH_SIZE", "16" if SMALL else "256"))   # reference :81 (per rank)
EPOCHS = 3                                                                  # reference :82
HVD_NP = int(os.environ.get("HVD_NP", "2"))
ARCH = default_arch()
DECODE = decode_mode()   # WORKSHOP_DECODE=gpu: nvJPEG + our resize kernel instead of CPU decode workers

cols_to_keep = ["content", "label_idx"]
train_df = catalog.table(f"{database_name}.silver_train").select(cols_to_keep)
val_df = catalog.table(f"{database_name}.silver_val").select(cols_to_keep)
num_classes = train_df.select("label_idx").distinct().count()

session.fs.rm(session.cache_dir, recurse=True)                             # reference :137
converter_train = make_converter(train_df, session.cache_dir)               # reference :140
converter_val = make_converter(val_df, session.cache_dir)
train_size, val_size = len(converter_train), len(converter_val)
print(f"train: {train_size}, val: {val_size}")
tracking.set_experiment(f"/Users/{user}/distributed_dl_workshop")
tracking_uri = tracking.get_tracking_uri()


def train_and_evaluate_hvd():
    """One rank = one process = one GPU (reference :282-375)."""
    hvd.init()                                                                               # :283
    tracking.set_tracking_uri(tracking_uri)                                                  # :286-288
    model = build_model(IMG_HEIGHT, IMG_WIDTH, IMG_CHANNELS, num_classes, arch=ARCH, batch_size=BATCH_SIZE)  # :298
    optimizer = optim.Adam(learning_rate=0.001 * hvd.size())                                 # :301  LR x world size
    optimizer = hvd.DistributedOptimizer(optimizer)                                          # :302
    callbacks = [                                                                            # :304-322 (and USED here)
        hvd.callbacks.BroadcastGlobalVariablesCallback(0),
        hvd.callbacks.MetricAverageCallback(),
        hvd.callbacks.LearningRateWarmupCallback(initial_lr=0.001 * hvd.size(), warmup_epochs=5, verbose=1),
        ReduceLROnPlateau(monitor="val_loss", patience=10, verbose=1),
    ]
    trainer = Trainer(model).compile(optimizer=optimizer, loss="sparse_categorical_crossentropy",
                                     metrics=["accuracy"])                                   # :325-328
    with converter_train.make_dataset(batch_size=BATCH_SIZE, cur_shard=hvd.rank(), shard_count=hvd.size(),
                                      image_size=(IMG_HEIGHT, IMG_WIDTH), decode=DECODE) as train_ds, \
         converter_val.make_dataset(batch_size=BATCH_SIZE, cur_shard=hvd.rank(), shard_count=hvd.size(),
                                    image_size=(IMG_HEIGHT, IMG_WIDTH), decode=DECODE) as val_ds:               # :332-337
        steps_per_epoch = max(1, train_size // (BATCH_SIZE * hvd.size()))                    # :350
        validation_steps = max(1, val_size // (BATCH_SIZE * hvd.size()))                     # :351
        hist = trainer.fit(train_ds, steps_per_epoch=steps_per_epoch, epochs=EPOCHS, verbose=1,
                           validation_data=val_ds, validation_steps=validation_steps, callbacks=callbacks)
    val_loss, val_accuracy = hist.history["val_loss"][-1], hist.history["val_accuracy"][-1]
    if hvd.rank() == 0:                                                                      # :361 log only from worker 0
        with tracking.start_run(run_id=active_run_uuid):
            tracking.log_params({"epochs": EPOCHS, "batch_size": BATCH_SIZE})
            tracking.log_metrics({"val_loss": val_loss, "val_accuracy": val_accuracy})
            tracking.keras.log_model(trainer, "model")
    return val_loss, val_accuracy                                                            # :375


# -- test on the driver only (np=-1), then distributed (reference :391-417)
with tracking.start_run(run_name="horovod_driver") as run:
    active_run_uuid = run.info.run_id
    print("driver-only:", Runner(np=-1, driver_log_verbosity="all").run(train_and_evaluate_hvd))
tracking.end_run()

with tracking.start_run(run_name="horovod_distributed") as run:
    active_run_uuid = run.info.run_id
    print(f"np={HVD_NP}:", Runner(np=HVD_NP, driver_log_verbosity="all").run(train_and_evaluate_hvd))
tracking.end_run()

converter_train.delete()                                                                     # :425-426
converter_val.delete()
trained_model = tracking.keras.load_model(f"runs:/{run.info.run_id}/model")                  # :438
trained_model.summary()
