from .coords import (cluster_coord, compare_coordinates, find_com, find_coord_clusters,
                     get_intensities, get_lengthscale_constraints, get_nn_distances,
                     get_nn_distances_, grid2xy, imcoordgrid, map_bonds, peak_refinement,
                     remove_edge_coord, subimg_trajectories, transform_coordinates)
from .graphx import (Graph, Node, filter_subgraphs, filter_subgraphs_, find_cycle_clusters,
                     find_cycles, get_interatomic_r, plot_graph)
from .img import (FFTmask, FFTsub, crop_borders, cv_thresh, extract_patches, extract_patches_,
                  extract_patches_and_spectra, extract_random_subimages, extract_subimages,
                  extract_subimages_cuda, filter_cells, filter_cells_, get_coord_grid,
                  get_imgstack, imcrop_randcoord, imcrop_randpx, img_pad, img_resize, threshImg)
from .imgen import (MakeAtom, create_atom_mask_pair, create_lattice_mask,
                    create_multiclass_lattice_mask, create_multiclass_lattice_mask_)
from .nn import (average_weights, get_downsample_factor, get_nb_classes, gpu_usage_map,
                 mock_forward, reset_bnorm, sample_weights, set_train_rng, weights_init)
from .preproc import (array2list, check_image_dims, check_signal_dims, create_batches,
                      get_array_memsize,
                      init_dataloader, init_dataloaders, init_fcnn_dataloaders,
                      init_imspec_dataloaders, num_classes_from_labels, preprocess_denoiser_data,
                      prepare_gp_input, preprocess_training_cls_data, preprocess_training_reg_data,
                      preprocess_training_image_data, preprocess_training_imspec_data,
                      shard_batches, torch_format_image, torch_format_spectra)
